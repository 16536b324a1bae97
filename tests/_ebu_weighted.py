"""The weighted EBU R128 restatement (tests/_ebu_weighted.cc): Ebu_r128_proc for 1..32 channels per instance with caller-given
channel weights, the oracle of b200m_ebu_create_weighted / b200m_r128_create_weighted.

The C++ source is compiled on first use into a private temporary directory (the tree may be read-only) with the reference's float
flags, the same ones oracle/Makefile uses for the CPU oracles: SSE2 arithmetic, no FMA contraction.  The compiler is $CXX, else g++.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "_ebu_weighted.cc")
FLAGS = ["-msse", "-msse2", "-mfpmath=sse", "-fomit-frame-pointer", "-O3", "-fno-finite-math-only", "-DNDEBUG"]
_v = C.c_void_p
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="b200m_ebu_weighted_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libebu_weighted.so")
        cxx = os.environ.get("CXX") or "g++"
        p = subprocess.run([cxx, *FLAGS, "-fPIC", "-shared", "-o", so, SRC, "-lm"], capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("compiling %s failed:\n%s" % (SRC, p.stderr))
        L = C.CDLL(so)
        for name, res, args in (("ew_create", _v, [C.c_int, C.c_int, _v, C.c_float]), ("ew_destroy", None, [_v]),
                                ("ew_integr", None, [_v, C.c_int, C.c_int]), ("ew_reset", None, [_v, C.c_int]),
                                ("ew_process", None, [_v, _v, C.c_size_t, C.c_int]), ("ew_read", None, [_v, _v]),
                                ("ew_hist", None, [_v, C.c_int, _v, _v, _v])):
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(_v)


class Ebu:
    """n_inst weighted Ebu_r128_proc instances; the interface of tests/_oracle.py's Ebu (integr, reset, process, read, hist)"""

    def __init__(self, n_inst, gains, fsamp=48000.0):
        self.L = lib()
        self.gains = np.ascontiguousarray(gains, np.float32).ravel()
        self.n, self.nchan = n_inst, self.gains.size
        self.h = self.L.ew_create(n_inst, self.nchan, _ptr(self.gains), fsamp)
        assert self.h, "1..32 channels"

    def __del__(self):
        if getattr(self, "h", None):
            self.L.ew_destroy(self.h)
            self.h = None

    def integr(self, cmd, inst=-1):
        self.L.ew_integr(self.h, inst, {"pause": 0, "start": 1, "reset": 2}[cmd])

    def reset(self, inst=-1):
        self.L.ew_reset(self.h, inst)

    def process(self, x):
        assert x.dtype == np.float32 and x.flags.c_contiguous and x.shape[0] == self.n * self.nchan
        self.L.ew_process(self.h, _ptr(x), x.shape[1], x.shape[1])

    def read(self):
        out = np.empty((self.n, 9), np.float32)
        self.L.ew_read(self.h, _ptr(out))
        return out

    def hist(self, inst):
        hm = np.empty(751, np.int32); hs = np.empty(751, np.int32); c = np.empty(4, np.int32)
        self.L.ew_hist(self.h, inst, _ptr(hm), _ptr(hs), _ptr(c))
        return hm, hs, c
