"""ctypes binding of libb2kin.so (the C ABI declared in include/b2kin.h).

There is no CPU fallback: if the CUDA library has not been built, or no CUDA device is
present when a compute entry point is called, this raises -- loudly -- instead of silently
computing on the host.  PyTorch is used only for device buffers and streams.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# B2K_LIB points the binding at another build of the same library (kernel experiments: scripts/ik_occ.sh)
LIB_PATH = os.environ.get("B2K_LIB") or os.path.join(_HERE, "lib", "libb2kin.so")

F32, F64 = 0, 1
MAX_JOINTS = 10
MAX_QWIDTH = 16
LM_METHODS = {"chan": 0, "wampler": 1, "sugihara": 2}
SEM_CPP, SEM_PYTHON = 0, 1
IK_NR, IK_GN = 3, 4  # method codes of b2k_ik_lm beyond the three LM damping rules
OPS_INV, OPS_PINV = 0, 1  # inverse kinds of b2k_opspace

_lib = None

vp = C.c_void_p
i64 = C.c_int64
dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)

_PROTOS = {
    "b2k_last_error": (C.c_char_p, []),
    "b2k_version": (C.c_int, []),
    "b2k_chain_create": (C.c_int, [C.c_int, ip, ip, ip, ip, dp, dp, C.POINTER(vp)]),
    "b2k_chain_destroy": (C.c_int, [vp]),
    "b2k_chain_info": (C.c_int, [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "b2k_fkine": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, vp]),
    "b2k_fkine_frames": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, C.c_int, ip, ip, dp, vp, i64, vp]),
    "b2k_jacob0": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, vp, vp]),
    "b2k_jacobe": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, vp, vp]),
    "b2k_fkine_jacob0": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, vp, vp]),
    "b2k_fkine_jacobe": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, vp, vp]),
    "b2k_ik_lm": (C.c_int, [vp, C.c_int, vp, i64, vp, C.c_int, C.c_int, C.c_double, C.c_int, dp, C.c_double,
                            C.c_int, C.c_uint64, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]),
    "b2k_ikine_null": (C.c_int, [vp, C.c_int, vp, i64, vp, C.c_int, C.c_int, C.c_double, C.c_int, dp, C.c_double,
                                 C.c_int, C.c_uint64, C.c_int, C.c_double, C.c_double, C.c_double, dp, vp, vp, vp, vp, vp,
                                 vp]),
    "b2k_rne_create": (C.c_int, [C.c_int, C.c_int, dp, C.POINTER(vp)]),
    "b2k_rne_destroy": (C.c_int, [vp]),
    "b2k_rne": (C.c_int, [vp, C.c_int, vp, vp, vp, i64, dp, dp, vp, vp]),
    "b2k_rne_wrench": (C.c_int, [vp, C.c_int, vp, vp, vp, i64, dp, dp, vp, vp, vp]),
    "b2k_rne_codegen": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_char_p, i64, dp, C.c_int32, ip, ip]),
    "b2k_rne_spec_info": (C.c_int, [vp, C.c_int, C.c_int, dp, C.c_int, C.c_char_p, i64]),
    "b2k_rne_fdyn": (C.c_int, [vp, C.c_int, vp, vp, i64, C.c_double, dp, C.c_int, dp, vp, dp, dp, dp, C.c_double, C.c_double,
                               C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]),
    "b2k_tree_fdyn": (C.c_int, [vp, C.c_int, vp, vp, i64, C.c_double, dp, C.c_int, dp, vp, dp, dp, dp, C.c_double, C.c_double,
                               C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]),
    "b2k_tree_create": (C.c_int, [C.c_int, ip, ip, ip, ip, dp, dp, C.POINTER(vp)]),
    "b2k_tree_destroy": (C.c_int, [vp]),
    "b2k_tree_rne": (C.c_int, [vp, C.c_int, vp, vp, vp, i64, dp, vp, vp]),
    "b2k_tree_dyn": (C.c_int, [vp, C.c_int, C.c_int, vp, vp, vp, i64, dp, vp, vp]),
    "b2k_tree_codegen": (C.c_int, [vp, C.c_int, C.c_int, C.c_char_p, i64, dp, C.c_int32, ip, ip]),
    "b2k_tree_info": (C.c_int, [vp, C.c_int, C.c_int, dp, C.c_char_p, i64]),
    "b2k_rne_inertia": (C.c_int, [vp, C.c_int, vp, i64, vp, vp]),
    "b2k_rne_gravload": (C.c_int, [vp, C.c_int, vp, i64, dp, vp, vp]),
    "b2k_rne_itorque": (C.c_int, [vp, C.c_int, vp, vp, i64, vp, vp]),
    "b2k_rne_coriolis": (C.c_int, [vp, C.c_int, vp, vp, i64, vp, vp]),
    "b2k_rne_accel": (C.c_int, [vp, C.c_int, vp, vp, vp, i64, dp, vp, vp]),
    "b2k_gravjac": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, vp, vp]),
    "b2k_pay": (C.c_int, [vp, C.c_int, vp, i64, i64, vp, i64, C.c_int, vp, vp]),
    "b2k_pay_jacobian": (C.c_int, [C.c_int, C.c_int, vp, vp, i64, i64, vp, vp]),
    "b2k_paycap": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, i64, C.c_int, dp, vp, vp, vp]),
    "b2k_friction": (C.c_int, [C.c_int, C.c_int, dp, vp, i64, vp, vp]),
    "b2k_hessian": (C.c_int, [C.c_int, C.c_int, vp, i64, vp, vp]),
    "b2k_manipulability": (C.c_int, [C.c_int, C.c_int, vp, i64, C.c_uint32, vp, vp]),
    "b2k_manipulability_svd": (C.c_int, [C.c_int, C.c_int, vp, i64, C.c_uint32, C.c_int, vp, vp]),
    "b2k_jacob_dot": (C.c_int, [C.c_int, C.c_int, vp, vp, i64, vp, vp]),
    "b2k_jacobm": (C.c_int, [C.c_int, C.c_int, vp, i64, C.c_uint32, vp, vp]),
    "b2k_angle_axis": (C.c_int, [C.c_int, vp, vp, i64, i64, vp, vp]),
    "b2k_p_servo": (C.c_int, [C.c_int, vp, vp, i64, i64, dp, C.c_double, vp, vp, vp]),
    "b2k_jacob0_analytical": (C.c_int, [C.c_int, C.c_int, vp, vp, i64, C.c_int, vp, vp]),
    "b2k_opspace": (C.c_int, [C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp]),
    "b2k_opspace_xdd": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, vp, i64, vp, vp]),
    "b2k_ikine_6s": (C.c_int, [C.c_int, dp, dp, dp, vp, i64, C.c_int, ip, vp, vp, vp]),
    "b2k_p_servo_rpy": (C.c_int, [C.c_int, vp, vp, i64, i64, dp, C.c_double, vp, vp, vp]),
    "b2k_ctraj": (C.c_int, [C.c_int, dp, dp, vp, i64, vp, vp]),
    "b2k_mstraj": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64), ip, dp, dp, dp, dp, i64, vp, vp]),
    "b2k_jtraj": (C.c_int, [C.c_int, C.c_int, dp, dp, dp, dp, i64, vp, C.c_double, vp, vp, vp, vp]),
    "b2k_mtraj": (C.c_int, [C.c_int, C.c_int, C.c_int, dp, dp, dp, dp, dp, i64, vp, C.c_double, vp, vp, vp, dp, vp]),
    "b2k_host_alloc": (C.c_int, [C.POINTER(vp), i64]),
    "b2k_host_free": (C.c_int, [vp]),
    "b2k_fkine_jacob0_host": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, vp, C.c_int]),
    "b2k_fkine_host": (C.c_int, [vp, C.c_int, vp, i64, i64, dp, dp, vp, C.c_int]),
    "b2k_rne_host": (C.c_int, [vp, C.c_int, vp, vp, vp, i64, dp, dp, vp, C.c_int]),
    "b2k_rne_wrench_host": (C.c_int, [vp, C.c_int, vp, vp, vp, i64, dp, dp, vp, vp, C.c_int]),
    "b2k_launch_count": (C.c_int64, []),
    "b2k_set_variant": (C.c_int, [C.c_int]),
    "b2k_selftest_sincos": (C.c_int, [C.c_int, vp, i64, vp, vp, vp]),
}

EXPORTED_SYMBOLS = tuple(_PROTOS)


class B2KError(RuntimeError):
    pass


def lib():
    """Load libb2kin.so (once).  Raises ImportError with build instructions if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: the CUDA library is not built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (or `make -C robotics-toolbox-python_b200/csrc`). "
                "There is no CPU fallback."
            )
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int):
    """Translate a b2k_status into the exception class the reference would raise."""
    if rc == 0:
        return
    msg = lib().b2k_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    raise B2KError(msg)


def dptr(a):
    """Optional host fp64 array -> double* (None -> NULL)."""
    if a is None:
        return None
    return a.ctypes.data_as(dp)


def f64_or_none(a, shape):
    if a is None:
        return None
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
    if a.shape != shape:
        a = a.reshape(shape)
    return a


def launch_count() -> int:
    return int(lib().b2k_launch_count())


def set_variant(v: int):
    check(lib().b2k_set_variant(int(v)))


class _PinnedPool:
    """Recycles page-locked host blocks: cudaHostAlloc of a few hundred MB costs ~100 ms, so result arrays
    handed to numpy callers come from (and return to) this cache.  At most B2K_PINNED_CACHE_MB (default
    2048) of freed blocks are kept; anything beyond is released to the driver."""

    GRAN = 1 << 20

    def __init__(self):
        import threading

        self.free = {}  # rounded size -> [ptr values]
        self.cached = 0
        self.limit = int(os.environ.get("B2K_PINNED_CACHE_MB", "2048")) << 20
        self.mu = threading.Lock()

    def take(self, nbytes):
        size = max(self.GRAN, (nbytes + self.GRAN - 1) // self.GRAN * self.GRAN)
        with self.mu:
            lst = self.free.get(size)
            if lst:
                self.cached -= size
                return lst.pop(), size
        p = vp()
        check(lib().b2k_host_alloc(C.byref(p), size))
        return p.value, size

    def give(self, ptr, size):
        with self.mu:
            if self.cached + size <= self.limit:
                self.free.setdefault(size, []).append(ptr)
                self.cached += size
                return
        try:
            lib().b2k_host_free(vp(ptr))
        except Exception:
            pass


_pool = None


def pinned_empty(shape, dtype=np.float64, pooled=False):
    """A numpy array backed by page-locked host memory (cudaHostAlloc), so the host-buffer
    front ends move it at full PCIe / C2C bandwidth.  The memory is released (pooled=True: returned to
    the recycling cache) when the array and all views of it are garbage collected."""
    global _pool
    dtype = np.dtype(dtype)
    count = int(np.prod(shape))
    n = count * dtype.itemsize
    if pooled:
        if _pool is None:
            _pool = _PinnedPool()
        addr, size = _pool.take(max(n, 1))
    else:
        p = vp()
        check(lib().b2k_host_alloc(C.byref(p), max(n, 1)))
        addr, size = p.value, None

    class _Owner:
        def __init__(self, addr, size):
            self.addr, self.size = addr, size

        def __del__(self):
            try:
                if self.size is None:
                    lib().b2k_host_free(vp(self.addr))
                else:
                    _pool.give(self.addr, self.size)
            except Exception:
                pass

    buf = (C.c_char * max(n, 1)).from_address(addr)
    buf._owner = _Owner(addr, size)  # keep-alive chain: ndarray -> buf -> owner
    return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)


def host_result(shape, dtype):
    """Result array of a host-buffer call: pooled pinned memory once it is large enough for the copy
    bandwidth to matter (>= 1 MB), plain numpy memory otherwise."""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    if n >= (1 << 20):
        return pinned_empty(shape, dtype, pooled=True)
    return np.empty(shape, dtype=dtype)
