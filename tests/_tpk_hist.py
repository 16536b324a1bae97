"""The oracle of the true-peak / K-meter bank's histogram plane (b200m_tpk_hist_*): per channel, the reference build's TruePeakdsp and
Kmeterdsp (_oracle.TruePeak, _oracle.Kmeter, one private meter each) fed only that channel's frames, with the distribution of their
readings counted by tests/_tpk_hist.cc.

- True peak: each frame's reading is the largest of its four |out|, taken from _oracle.tp_upsample (the reference build's resampler,
  run over every frame the channel was fed so far; its outputs do not depend on how the frames are cut into calls).  After each
  block the oracle's TruePeak is read, and when every frame of the block is finite its p must equal the block's largest reading bit
  for bit: the frames are those of the reference's own trajectory.
- K-meter: before each block the meter's z1 z2 are copied from the oracle (Kmeter.peek) and tests/_tpk_hist.cc steps the copies over
  the block, counting each group's reading.  Then the oracle runs the block itself, and its z1 z2 must equal the copies' bit for bit.

The C++ source is compiled on first use into a private temporary directory (the tree may be read-only) with the reference's float
flags, as tests/_ppm_hist.py does.  The compiler is $CXX, else g++.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import _oracle as O
from _ppm_hist import BINS, EDGES, FLAGS, empty, limit

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "_tpk_hist.cc")
TP, KM = 1, 2
_v = C.c_void_p
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="b200m_tpk_hist_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libtpk_hist.so")
        cxx = os.environ.get("CXX") or "g++"
        p = subprocess.run([cxx, *FLAGS, "-fPIC", "-shared", "-o", so, SRC, "-lm"], capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("compiling %s failed:\n%s" % (SRC, p.stderr))
        L = C.CDLL(so)
        L.th_count.restype = None
        L.th_count.argtypes = [_v, C.c_int, C.c_float, _v, _v, _v]
        L.th_km_run.restype = None
        L.th_km_run.argtypes = [C.c_float, C.c_float, _v, _v, C.c_int, _v, _v, _v]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(_v)


def count(u, lim, counts, stats):
    """count the readings u (float32, any order of finite and non-finite) into one row: counts uint64 [242], stats STATS [1]"""
    u = np.ascontiguousarray(u, np.float32)
    lib().th_count(_ptr(u), u.size, np.float32(lim), _ptr(EDGES), _ptr(counts), _ptr(stats))


def frame_readings(up):
    """the true-peak readings of frames whose 4x-oversampled outputs are `up` (float32 [4 n]): the largest |out| of each frame, NaN
    where one of them is not finite"""
    a = np.abs(np.asarray(up, np.float32).reshape(-1, 4))
    u = a.max(axis=1)
    u[~np.isfinite(a).all(axis=1)] = np.nan
    return u


class TpkHist:
    """n channels of private reference meters (flags TP / KM / both) with the distribution of their readings"""

    def __init__(self, n, fsamp=48000.0, flags=TP | KM, tp_limit_db=-1.0, km_limit_db=-10.0, oracle="best"):
        self.n, self.fs, self.flags, self.oracle = n, float(fsamp), flags, oracle
        self.tp = [O.TruePeak(1, fsamp, oracle) for _ in range(n)] if flags & TP else None
        self.km = [O.Kmeter(1, fsamp, oracle) for _ in range(n)] if flags & KM else None
        self.omega = np.float32(self.km[0].coeffs()[0]) if self.km else None
        self.fed = [np.zeros(0, np.float32) for _ in range(n)]
        self.tp_p = np.zeros(n, np.float32)                 # the last read()'s p of each channel
        self.clear_hist(tp_limit_db, km_limit_db)

    def clear_hist(self, tp_limit_db=None, km_limit_db=None):
        """what b200m_tpk_hist_enable does to the rows (and the limits, when given)"""
        self.rows = {q: (np.zeros((self.n, BINS), np.uint64), empty(self.n)) for q in ("tp", "km")}
        if tp_limit_db is not None:
            self.tp_lim = limit(tp_limit_db)
        if km_limit_db is not None:
            self.km_lim = limit(km_limit_db)

    def reset(self, tp=True, km=True):
        """b200m_tpk_reset of every channel (tp and km), or b200m_tpk_reset_kmeter (km only): the meters' reset(), the rows untouched"""
        for i in range(self.n):
            if tp and self.tp:
                self.tp[i].reset()
            if km and self.km:
                self.km[i].reset()

    def clear(self, i):
        """b200m_tpk_clear of channel i with the plane on: fresh meters and empty rows"""
        if self.tp:
            self.tp[i] = O.TruePeak(1, self.fs, self.oracle)
        if self.km:
            self.km[i] = O.Kmeter(1, self.fs, self.oracle)
        self.fed[i] = np.zeros(0, np.float32)
        for c, s in self.rows.values():
            c[i] = 0
            s[i] = empty(1)[0]

    def process(self, x, lengths=None, read=True):
        """one process() block of every channel over its first lengths[i] frames (None: all); read: read() every true-peak meter
        after it and check the block's largest finite reading against p"""
        x = np.ascontiguousarray(x, np.float32)
        assert x.ndim == 2 and x.shape[0] == self.n
        ln = np.full(self.n, x.shape[1]) if lengths is None else np.asarray(lengths)
        for i in range(self.n):
            L = int(ln[i])
            if L == 0:
                continue
            xi = np.ascontiguousarray(x[i:i + 1, :L])
            if self.tp:
                before = self.fed[i].size
                self.fed[i] = np.concatenate([self.fed[i], xi[0]])
                u = frame_readings(O.tp_upsample(self.fed[i], self.fs, 1024, self.oracle)[4 * before:])
                c, s = self.rows["tp"]
                st = s[i:i + 1].copy()
                count(u, self.tp_lim, c[i], st)
                s[i] = st[0]
                self.tp[i].process(xi)
                if read:
                    self.tp_p[i] = self.tp[i].read()[1][0]
                    if np.isfinite(u).all():
                        assert u.max().view(np.uint32) == self.tp_p[i].view(np.uint32), "the frames left the reference's trajectory"
            if self.km:
                z = np.ascontiguousarray(self.km[i].peek()[0, :2])
                c, s = self.rows["km"]
                st = s[i:i + 1].copy()
                lib().th_km_run(self.omega, self.km_lim, _ptr(z), _ptr(xi), L, _ptr(EDGES), _ptr(c[i]), _ptr(st))
                s[i] = st[0]
                self.km[i].process(xi)
                assert np.array_equal(self.km[i].peek()[0, :2].view(np.uint32), z.view(np.uint32)), "the K-meter copy left the oracle's trajectory"

    def hist(self):
        """(tp_counts, tp_stats, km_counts, km_stats) as TruePeakKmeter.hist returns them, None for an absent meter"""
        out = []
        for q, f in (("tp", TP), ("km", KM)):
            c, s = self.rows[q]
            out += [c.astype(np.int64), s.copy()] if self.flags & f else [None, None]
        return tuple(out)
