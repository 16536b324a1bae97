"""The oracle of the needle-meter bank's histogram plane (b200m_ppm_hist_*): an _oracle.Needle bank (the reference build, or the
port) whose per-group readings are counted by tests/_ppm_hist.cc on copies of its meter states.

Before each block, every meter's z1 z2 m res is copied from the oracle (Needle.peek) and tests/_ppm_hist.cc steps the copies over
the block, counting each group's reading with the rules the bank documents.  Then the oracle runs the block itself, and its states
must equal the copies' bit for bit: the counts are those of the reference build's own needles.

The C++ source is compiled on first use into a private temporary directory (the tree may be read-only) with the reference's float
flags, as tests/_cor_hist.py does.  The compiler is $CXX, else g++.
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
SRC = os.path.join(HERE, "_ppm_hist.cc")
FLAGS = ["-msse", "-msse2", "-mfpmath=sse", "-fomit-frame-pointer", "-O3", "-fno-finite-math-only", "-DNDEBUG"]
BINS = 242
# the bin edges, computed independently of the library: float64 10^((-80 + 0.5 k) / 20) rounded to float32
EDGES = (10.0 ** ((-80.0 + 0.5 * np.arange(BINS - 1)) / 20.0)).astype(np.float32)
STATS = np.dtype([("nonfinite", "<u8"), ("over_groups", "<u8"), ("overs", "<u8"), ("longest_over", "<u8"), ("run", "<u8"),
                  ("peak", "<f4"), ("pad", "<u4")])
_v = C.c_void_p
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="b200m_ppm_hist_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libppm_hist.so")
        cxx = os.environ.get("CXX") or "g++"
        p = subprocess.run([cxx, *FLAGS, "-fPIC", "-shared", "-o", so, SRC, "-lm"], capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("compiling %s failed:\n%s" % (SRC, p.stderr))
        L = C.CDLL(so)
        L.ph_run.restype = None
        L.ph_run.argtypes = [C.c_int, C.c_int, _v, C.c_float, C.c_float, C.c_float, _v, _v, C.c_size_t, C.c_int, _v, _v, _v]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(_v)


def limit(limit_db):
    """the bank's over limit L = (float) 10^(limit_db / 20), computed in double"""
    with np.errstate(over="ignore"):
        return np.float32(10.0 ** (float(limit_db) / 20.0))


def empty(nm):
    """nm rows of cleared statistics: zero, peak -inf"""
    s = np.zeros(nm, STATS)
    s["peak"] = -np.inf
    return s


class Needle:
    """an oracle needle bank (_oracle.Needle: kind 0 VU / 1 IEC I / 2 IEC II on n mono rows, 3 M/S on n pairs) with the histogram
    and statistics of its per-group readings"""

    def __init__(self, n, kind, fsamp=48000.0, limit_db=0.0, oracle="best"):
        self.o = O.Needle(n, kind, fsamp, oracle)
        self.n, self.kind, self.nm = n, kind, self.o.nm
        self.w = np.ascontiguousarray(self.o.coeffs(), np.float32)
        self.lim = limit(limit_db)
        self.db = (-6.0, -6.0)
        self.counts = np.zeros((self.nm, BINS), np.uint64)
        self.stats = empty(self.nm)

    def set_gain(self, db_m, db_s):
        self.o.set_gain(db_m, db_s)
        self.db = (db_m, db_s)

    def process(self, x, nthreads=1):
        x = np.ascontiguousarray(x, np.float32)
        assert x.ndim == 2 and x.shape[0] == self.nm
        nfram = x.shape[1]
        s = np.ascontiguousarray(self.o.peek())
        lib().ph_run(self.n, self.kind, _ptr(self.w), self.lim, self.db[0], self.db[1], _ptr(s), _ptr(x), max(nfram, 1), nfram,
                     _ptr(EDGES), _ptr(self.counts), _ptr(self.stats))
        self.o.process(x, nthreads)
        assert np.array_equal(self.o.peek().view(np.uint32), s.view(np.uint32)), "the copied meters left the oracle's trajectory"

    def clear_hist(self, limit_db=None):
        """what b200m_ppm_hist_enable does to the counts and statistics (and the limit, when given)"""
        self.counts[:] = 0
        self.stats = empty(self.nm)
        if limit_db is not None:
            self.lim = limit(limit_db)

    def hist(self):
        """(counts int64 [nm, 242], stats [nm]), as NeedleMeters.hist of the bank returns them"""
        return self.counts.astype(np.int64), self.stats.copy()

    def read(self):
        return self.o.read()

    def peek(self):
        return self.o.peek()
