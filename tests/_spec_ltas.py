"""The oracle of the spectrum bank's long-term average spectrum (b200m_spec_ltas_*): an _oracle.Spectr30 bank (the reference build,
or the port) whose per-frame band power is summed by tests/_spec_ltas.cc on copies of its filter states.

Before each block, every instance's filter state is copied from the oracle (Spectr30.state) and tests/_spec_ltas.cc runs the 30
band cascades on the copies over the block, adding each finite float s = v * v to the band's double sum in frame order and counting
it.  Then the oracle runs the block itself, and its filter states must equal the copies' bit for bit: the sums are the LTAS of the
oracle's own per-frame power, with the rule the bank documents (a non-finite s adds nothing and is not counted).

The C++ source is compiled on first use into a private temporary directory (the tree may be read-only) with the reference's float
flags, as tests/_ebu_weighted.py does.  The compiler is $CXX, else g++.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import _oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "_spec_ltas.cc")
FLAGS = ["-msse", "-msse2", "-mfpmath=sse", "-fomit-frame-pointer", "-O3", "-fno-finite-math-only", "-DNDEBUG"]
_v = C.c_void_p
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="b200m_spec_ltas_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libspec_ltas.so")
        cxx = os.environ.get("CXX") or "g++"
        p = subprocess.run([cxx, *FLAGS, "-fPIC", "-shared", "-o", so, SRC, "-lm"], capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("compiling %s failed:\n%s" % (SRC, p.stderr))
        L = C.CDLL(so)
        L.sl_run.restype = None
        L.sl_run.argtypes = [C.c_int, C.c_int, _v, _v, _v, C.c_size_t, _v, _v, _v, _v]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(_v)


class Spectr30:
    """n_inst oracle spectr30 instances run in lock step (_oracle.Spectr30) with the LTAS of their per-frame band power"""

    def __init__(self, n_inst, nchan=2, rate=48000.0, kind="best"):
        self.o = O.Spectr30(n_inst, nchan, rate, kind)
        self.n, self.nchan = n_inst, nchan
        self.W = np.ascontiguousarray(self.o.coeffs())
        self.frames = np.zeros(n_inst, np.int64)
        self.sums = np.zeros((n_inst, 30), np.float64)
        self.counts = np.zeros((n_inst, 30), np.uint64)

    def _z(self):
        return np.ascontiguousarray(np.stack([self.o.state(i)[0] for i in range(self.n)]))

    def process(self, x, speed=1.0, reset=-4.0, nthreads=1):
        x = np.ascontiguousarray(x, np.float32)
        assert x.ndim == 2 and x.shape[0] == self.n * self.nchan
        nfram = x.shape[1]
        z = self._z()
        ln = np.full(self.n, nfram, np.int32)
        lib().sl_run(self.n, self.nchan, _ptr(self.W), _ptr(z), _ptr(x), max(nfram, 1), _ptr(ln), _ptr(self.frames),
                     _ptr(self.sums), _ptr(self.counts))
        self.o.process(x, speed, reset, nthreads)
        assert np.array_equal(self._z().view(np.uint64), z.view(np.uint64)), "the copied cascades left the oracle's trajectory"
        self.frames += nfram

    def clear_ltas(self):
        """what b200m_spec_ltas_enable does to the sums and counts"""
        self.sums[:] = 0
        self.counts[:] = 0

    def ltas(self):
        """(sums float64 [n_inst, 30], counts int64 [n_inst, 30]), as Spectr30.ltas of the bank returns them"""
        return self.sums.copy(), self.counts.astype(np.int64)

    def read(self):
        return self.o.read()

    def state(self, inst):
        return self.o.state(inst)
