"""Minimal stand-ins for spatialmath's SE3 and SE2 (spatialmath-python is not a dependency here).

``ETS.fkine`` in the reference wraps every pose of a trajectory into its own SE3 object
(reference ETS.py:1013-1015) -- O(N) Python objects, which for a 1M-row batch costs far more
than the kinematics.  These containers keep the batch as one (N,4,4) / (N,3,3) array and only expose the
few accessors the hot path's callers use (.A, .t, .R, len, indexing, iteration)."""
from __future__ import annotations

import numpy as np


class _SEn:
    _D = 4  # side of the homogeneous matrix

    def __init__(self, A):
        A = getattr(A, "A", A)
        A = np.asarray(A)
        D = self._D
        if A.shape[-2:] != (D, D):
            raise ValueError(f"{type(self).__name__} needs ({D},{D}) or (N,{D},{D}) data")
        self._A = A.reshape(-1, D, D)
        self._single = A.ndim == 2

    @property
    def A(self):
        return self._A[0] if self._single else self._A

    @property
    def t(self):
        return self.A[..., : self._D - 1, self._D - 1]

    @property
    def R(self):
        return self.A[..., : self._D - 1, : self._D - 1]

    def __len__(self):
        return self._A.shape[0]

    def __getitem__(self, i):
        return type(self)(self._A[i])

    def __iter__(self):
        for i in range(self._A.shape[0]):
            yield type(self)(self._A[i])

    def __repr__(self):
        return f"{type(self).__name__}(n={len(self)})\n{self.A}"


class SE3(_SEn):
    _D = 4


class SE2(_SEn):
    """Planar poses: .t is (...,2), .R is (...,2,2)."""

    _D = 3
