"""Two-link planar arm (reference models/ETS/Planar2.py, restated): R . tx(1) . R . tx(1), qz = [0, 0]."""
from ..ET import ET2
from ..Robot2 import Robot2


class Planar2(Robot2):
    def __init__(self):
        a1 = a2 = 1.0
        super().__init__(ET2.R() * ET2.tx(a1) * ET2.R() * ET2.tx(a2), name="Planar2")
        self.addconfiguration("qz", [0.0, 0.0])
