"""Constant tables of the benchmark robots (SURVEY 8a row M), restated from the reference:

    Panda    ETS  reference models/ETS/Panda.py:28-64
    Puma560  DH   reference models/DH/Puma560.py:87-201
    UR10     DH   reference models/DH/UR10.py:52-118
    PandaMDH DH   reference models/DH/Panda.py:36-173  (modified DH, cross-check of the ETS model)
    Planar2  ETS2 reference models/ETS/Planar2.py       (planar two-link arm)
"""
from .Panda import Panda  # noqa: F401
from .Planar2 import Planar2  # noqa: F401
from .PandaMDH import PandaMDH  # noqa: F401
from .Puma560 import Puma560  # noqa: F401
from .UR10 import UR10  # noqa: F401


class ETS:  # namespace parity with rtb.models.ETS.Panda
    Panda = Panda
    Planar2 = Planar2


class DH:  # namespace parity with rtb.models.DH.*
    Puma560 = Puma560
    UR10 = UR10
    Panda = PandaMDH
