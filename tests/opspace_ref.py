"""Restatement of the reference's operational-space dynamics -- DynamicsMixin inertia_x / coriolis_x / gravload_x /
accel_x (robot/Dynamics.py, between gravload and itorque) -- per row with numpy's inv / pinv, over the oracle's dyn_*
loops and its jacob0_analytical.  Test infrastructure only: test_opspace_cpu.py pins it by identities (equation of
motion, Penrose conditions), test_gpu_opspace.py checks the device against it.

`chain` is an oracle Chain of the robot's kinematics (what jacob0_analytical sees); rne_fn / rne_nofriction_fn /
gravity follow the conventions of the oracle's dyn_* functions.
"""
import numpy as np

from oracle import oracle as orc


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def ja(chain, q, representation="rpy/xyz"):
    q = np.atleast_2d(_f64(q))
    return orc.jacob0_analytical(chain.fkine(q), chain.jacob0(q), representation)


def jad(chain, q, qd, representation="rpy/xyz", h=1e-6):
    """ETS.jacob0_dot(q, qd, representation=...): the central difference of Ja along qd"""
    q, qd = np.atleast_2d(_f64(q)), np.atleast_2d(_f64(qd))
    return (ja(chain, q + h * qd, representation) - ja(chain, q - h * qd, representation)) / (2 * h)


def ji(Ja, pinv=False):
    return np.linalg.pinv(Ja) if pinv else np.linalg.inv(Ja)


def inertia_x(rne_fn, chain, n, q, pinv=False, representation="rpy/xyz"):
    """Mx = Ji^T M Ji"""
    Ji = ji(ja(chain, q, representation), pinv)
    return Ji.transpose(0, 2, 1) @ orc.dyn_inertia(rne_fn, n, q) @ Ji


def gravload_x(rne_fn, chain, n, q, gravity, pinv=False, representation="rpy/xyz"):
    """Gx = Ji^T G"""
    Ji = ji(ja(chain, q, representation), pinv)
    return np.einsum("kia,ki->ka", Ji, orc.dyn_gravload(rne_fn, n, q, gravity))


def coriolis_x(rne_fn, rne_nofriction_fn, chain, n, q, qd, pinv=False, representation="rpy/xyz", h=1e-6):
    """Cx = Ji^T C Ji - Mx Jad Ji (h: the difference step of Jad; ETS.jacob0_dot takes 1e-3 in fp32)"""
    Ji = ji(ja(chain, q, representation), pinv)
    JiT = Ji.transpose(0, 2, 1)
    Mx = JiT @ orc.dyn_inertia(rne_fn, n, q) @ Ji
    return JiT @ orc.dyn_coriolis(rne_nofriction_fn, n, q, qd) @ Ji - Mx @ jad(chain, q, qd, representation, h) @ Ji


def accel_x(rne_fn, chain, n, q, xd, wrench, gravity, pinv=False, representation="rpy/xyz", h=1e-6):
    """qd = Ji xd, qdd = accel(q, qd, Ja^T w), xdd = Ja qdd + Jad qd"""
    q = np.atleast_2d(_f64(q))
    xd, wrench = (np.broadcast_to(np.atleast_2d(_f64(x)), (q.shape[0], 6)) for x in (xd, wrench))
    Ja = ja(chain, q, representation)
    Ji = ji(Ja, pinv)
    qd = np.einsum("kij,kj->ki", Ji, xd)
    tau = np.einsum("kri,kr->ki", Ja, wrench)
    qdd = orc.dyn_accel(rne_fn, n, q, qd, tau, gravity)
    return np.einsum("kri,ki->kr", Ja, qdd) + np.einsum("kri,ki->kr", jad(chain, q, qd, representation, h), qd)
