"""TEST-ONLY: the oracle with every channel's noise-floor filters readable.  oracle/pyoracle.Oracle keeps mag_lp / mag_nf
inside its channel records; tests/hostsim/oracle_noise_floor.c compiles the unchanged oracle source together with one
reader of them, and Oracle here is pyoracle's Oracle running on that build."""
import ctypes as C
import os
import subprocess
import tempfile
import numpy as np
from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    """the build of the oracle with vo_noise_floor, its functions typed as pyoracle types the plain build's"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="oracle_nf_"), "liboracle_nf.so")
        subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w", "-o", so,
                               os.path.join(_HERE, "hostsim", "oracle_noise_floor.c"), "-lm"])
        L = C.CDLL(so)
        for name, f in vars(po.lib()).items():          # the functions pyoracle has typed (ctypes caches them by name)
            if isinstance(f, C._CFuncPtr):
                g = getattr(L, name)
                g.argtypes, g.restype = f.argtypes, f.restype
        L.vo_noise_floor.argtypes = [C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


class Oracle(po.Oracle):
    """po.Oracle whose context lives in the build above, plus noise_floor()"""

    def __init__(self, *args, **kw):
        plain = po._LIB
        po._LIB = lib()                                   # the base constructor takes its library from pyoracle.lib()
        try:
            super().__init__(*args, **kw)
        finally:
            po._LIB = plain

    def noise_floor(self):
        """every channel's noise-floor filters as they stand now, [n_channels][2] float32: mag_lp, mag_nf"""
        a = np.zeros((self.n_channels, 2), np.float32)
        self.L.vo_noise_floor(self.h, a.ctypes.data)
        return a
