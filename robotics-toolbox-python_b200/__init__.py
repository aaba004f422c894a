"""b2kin -- H100-native batched robot kinematics & dynamics.

A drop-in for ONE hot path of petercorke/robotics-toolbox-python: serial-chain forward
kinematics, geometric Jacobians, DH recursive Newton-Euler and Levenberg-Marquardt IK over an
(N, n) batch of joint configurations, computed by hand-written sm_90a CUDA kernels behind the
C ABI in include/b2kin.h.  The classes keep the reference's names (ET, ETS, DHRobot, Robot,
IKSolution, IK_LM, models.*).  The directory name is not a Python identifier; import it as

    import b2kin as rtb            # the alias module at the repository root

There is no CPU fallback in this package.
"""
from . import _lib  # noqa: F401
from ._lib import B2KError, launch_count, pinned_empty  # noqa: F401
from ._se3 import SE2, SE3  # noqa: F401
from .ET import ET, ET2  # noqa: F401
from .IK import IK_GN, IK_LM, IK_NR, IK_QP, IKSolution  # noqa: F401
from .ETS import ETS, ETS2  # noqa: F401
from .DHLink import DHLink, PrismaticDH, PrismaticMDH, RevoluteDH, RevoluteMDH  # noqa: F401
from .DHRobot import DHRobot  # noqa: F401
from .Robot import ERobot, Link, Robot  # noqa: F401
from .Robot2 import Link2, Robot2  # noqa: F401
from . import models  # noqa: F401
from . import dist  # noqa: F401
from . import trajectory  # noqa: F401
from .trajectory import Trajectory, ctraj, jtraj, lspb, mstraj, mtraj, quintic, trapezoidal  # noqa: F401
from .p_servo import angle_axis, p_servo  # noqa: F401



def rne_kernel_info(robot, op="rne", dtype="float64") -> str:
    """One line describing the kernel that serves `robot.<op>` (see DHRobot.rne_kernel_info)."""
    import numpy as _np

    return robot.rne_kernel_info(op, _np.dtype(dtype))


def rne_kernel_name(robot) -> str:
    return rne_kernel_info(robot).split(":")[0]


__version__ = "0.1.0"
