"""The oracle of the correlation bank's histogram plane (b200m_cor_hist_*): an _oracle.Stcorr bank (the reference build, or the
port) whose per-frame readings are counted by tests/_cor_hist.cc on copies of its filter states.

Before each block, every pair's five states are copied from the oracle (Stcorr.peek) and tests/_cor_hist.cc steps the copies over
the block, counting each frame's reading in its bin and adding it to the pair's double sum when the gate passes.  Then the oracle
runs the block itself, and its states must equal the copies' bit for bit: the counts are those of the reference build's own
trajectory, with the rules the bank documents.

The C++ source is compiled on first use into a private temporary directory (the tree may be read-only) with the reference's float
flags, as tests/_spec_ltas.py does.  The compiler is $CXX, else g++.
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
SRC = os.path.join(HERE, "_cor_hist.cc")
FLAGS = ["-msse", "-msse2", "-mfpmath=sse", "-fomit-frame-pointer", "-O3", "-fno-finite-math-only", "-DNDEBUG"]
BINS = 200
_v = C.c_void_p
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="b200m_cor_hist_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libcor_hist.so")
        cxx = os.environ.get("CXX") or "g++"
        p = subprocess.run([cxx, *FLAGS, "-fPIC", "-shared", "-o", so, SRC, "-lm"], capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("compiling %s failed:\n%s" % (SRC, p.stderr))
        L = C.CDLL(so)
        L.ch_run.restype = None
        L.ch_run.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, _v, _v, C.c_size_t, C.c_int, _v, _v]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(_v)


def gate(gate_db):
    """the bank's threshold on zll + zrr: (float) (2 * 10^(gate_db / 10)), computed in double"""
    return np.float32(2.0 * 10.0 ** (float(gate_db) / 10.0))


class Stcorr:
    """n oracle Stcorrdsp pairs run in lock step (_oracle.Stcorr) with the histogram of their per-frame readings"""

    def __init__(self, n, fsamp=48000, flp=2e3, tcf=0.3, gate_db=-70.0, kind="best"):
        self.o = O.Stcorr(n, fsamp, flp, tcf, kind)
        self.n = n
        self.w = self.o.coeffs()
        self.thr = gate(gate_db)
        self.counts = np.zeros((n, BINS), np.uint64)
        self.sums = np.zeros(n, np.float64)

    def process(self, x, nthreads=1):
        x = np.ascontiguousarray(x, np.float32)
        assert x.ndim == 2 and x.shape[0] == 2 * self.n
        nfram = x.shape[1]
        s = np.ascontiguousarray(self.o.peek())
        lib().ch_run(self.n, self.w[0], self.w[1], self.thr, _ptr(s), _ptr(x), max(nfram, 1), nfram, _ptr(self.counts),
                     _ptr(self.sums))
        self.o.process(x, nthreads)
        assert np.array_equal(self.o.peek().view(np.uint32), s.view(np.uint32)), "the copied recurrences left the oracle's trajectory"

    def clear_hist(self, gate_db=None):
        """what b200m_cor_hist_enable does to the counts and sums (and the gate, when given)"""
        self.counts[:] = 0
        self.sums[:] = 0
        if gate_db is not None:
            self.thr = gate(gate_db)

    def hist(self):
        """(counts int64 [n, 200], sums float64 [n]), as Stcorrdsp.hist of the bank returns them"""
        return self.counts.astype(np.int64), self.sums.copy()

    def read(self):
        return self.o.read()

    def peek(self):
        return self.o.peek()
