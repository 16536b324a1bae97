"""ctypes loader for the CPU oracles (oracle/oracle_api.h).  TEST INFRASTRUCTURE ONLY.

`load("reference")` -> oracle/_ref/libmeters_ref.so (unmodified reference sources, built here by
oracle/Makefile and shipped prebuilt to the GPU box); `load("port")` -> oracle/liboracle_port.so
(this repo's CPU restatement).  `load("best")` prefers the reference build.
"""
import ctypes as C
import os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATHS = {
    "reference": os.path.join(ROOT, "oracle", "_ref", "libmeters_ref.so"),
    "port": os.path.join(ROOT, "oracle", "liboracle_port.so"),
}
_f = C.POINTER(C.c_float)
_d = C.POINTER(C.c_double)
_i = C.POINTER(C.c_int)
_v = C.c_void_p


def available(kind):
    return os.path.exists(PATHS[kind])


def _proto(lib):
    P = {
        "orc_kind": (C.c_char_p, []),
        "orc_hw_threads": (C.c_int, []),
        "orc_ebu_create": (_v, [C.c_int, C.c_int, C.c_float]),
        "orc_ebu_destroy": (None, [_v]),
        "orc_ebu_integr": (None, [_v, C.c_int, C.c_int]),
        "orc_ebu_reset": (None, [_v, C.c_int]),
        "orc_ebu_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_ebu_read": (None, [_v, _v]),
        "orc_ebu_hist": (None, [_v, C.c_int, _v, _v, _v]),
        "orc_ebu_coeffs": (None, [_v, _v]),
        "orc_ebu_state": (None, [_v, C.c_int, _v, _v, _v, _v]),
        "orc_ebu_hist_calc": (None, [_v, C.c_int, _v, C.c_int, _v]),
        "orc_r128_cycle": (None, [_v, _v, _v, C.c_size_t, C.c_int, C.c_int, C.c_int]),
        "orc_tp_create": (_v, [C.c_int, C.c_float]),
        "orc_tp_destroy": (None, [_v]),
        "orc_tp_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int, C.c_int]),
        "orc_tp_read": (None, [_v, _v, _v]),
        "orc_tp_peek": (None, [_v, _v, _v, _v, _v, _v]),
        "orc_tp_reset": (None, [_v, C.c_int]),
        "orc_tp_coeffs": (None, [_v, _v, _v]),
        "orc_tp_upsample": (None, [C.c_float, _v, C.c_int, C.c_int, _v]),
        "orc_km_create": (_v, [C.c_int, C.c_float]),
        "orc_km_destroy": (None, [_v]),
        "orc_km_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_km_read": (None, [_v, _v, _v]),
        "orc_km_peek": (None, [_v, _v]),
        "orc_km_reset": (None, [_v, C.c_int]),
        "orc_km_coeffs": (None, [_v, _v, _v]),
        "orc_ppm_create": (_v, [C.c_int, C.c_float, C.c_int]),
        "orc_ppm_destroy": (None, [_v]),
        "orc_ppm_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_ppm_read": (None, [_v, _v]),
        "orc_ppm_peek": (None, [_v, _v]),
        "orc_ppm_set_gain": (None, [_v, C.c_float, C.c_float]),
        "orc_ppm_coeffs": (None, [_v, _v]),
        "orc_ebuplug_create": (_v, [C.c_int, C.c_float, C.c_int]),
        "orc_ebuplug_destroy": (None, [_v]),
        "orc_ebuplug_run": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_ebuplug_read": (None, [_v, _v]),
        "orc_bim_create": (_v, [C.c_int, C.c_float]),
        "orc_bim_destroy": (None, [_v]),
        "orc_bim_mode": (None, [_v, C.c_int, C.c_int]),
        "orc_bim_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_bim_read": (None, [_v, C.c_int, _v, _v, _v, _v]),
        "orc_sdh_create": (_v, [C.c_int, C.c_float]),
        "orc_sdh_destroy": (None, [_v]),
        "orc_sdh_integrate": (None, [_v, C.c_int]),
        "orc_sdh_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_sdh_read": (None, [_v, C.c_int, _v, _v, _v, _v]),
        "orc_cor_create": (_v, [C.c_int, C.c_int, C.c_float, C.c_float]),
        "orc_cor_destroy": (None, [_v]),
        "orc_cor_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_cor_read": (None, [_v, _v]),
        "orc_cor_peek": (None, [_v, _v]),
        "orc_cor_coeffs": (None, [_v, _v]),
        "orc_spec_create": (_v, [C.c_int, C.c_int, C.c_double]),
        "orc_spec_destroy": (None, [_v]),
        "orc_spec_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_float, C.c_float, C.c_int]),
        "orc_spec_read": (None, [_v, _v]),
        "orc_spec_state": (None, [_v, C.c_int, _v, _v, _v]),
        "orc_spec_coeffs": (None, [_v, _v]),
        "orc_dr14_create": (_v, [C.c_int, C.c_int, C.c_double, C.c_int]),
        "orc_dr14_destroy": (None, [_v]),
        "orc_dr14_process": (None, [_v, _v, C.c_size_t, C.c_int, C.c_int]),
        "orc_dr14_reset": (None, [_v]),
        "orc_dr14_read": (None, [_v, _v]),
        "orc_pw_create": (_v, [C.c_int, C.c_int, C.c_double]),
        "orc_pw_destroy": (None, [_v]),
        "orc_pw_set_mode": (None, [_v, C.c_int]),
        "orc_pw_process": (C.c_int, [_v, _v, C.c_size_t, C.c_int, C.c_float, C.c_int]),
        "orc_pw_read": (None, [_v, _v, _v, _v]),
        "orc_pw_raw": (None, [_v, C.c_int, _v, _v, _v, _v]),
        "orc_log10f_check": (C.c_longlong, [C.c_uint32, C.c_uint32, _v, C.c_int, _v]),
        "orc_cpu_info": (C.c_int, [_v, _v, _v]),
        "orc_r128_bench": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _v]),
    }
    # a prebuilt reference library from before an entry was added lacks it: the other entries stay usable, and
    # exports() says which ones the library has
    lib.orc_exports = set()
    for name, (res, args) in P.items():
        fn = getattr(lib, name, None)
        if fn is None:
            continue
        fn.restype = res
        fn.argtypes = args
        lib.orc_exports.add(name)
    return lib


_cache = {}


def load(kind="best"):
    if kind == "best":
        kind = "reference" if available("reference") else "port"
    if kind not in _cache:
        _cache[kind] = _proto(C.CDLL(PATHS[kind]))
    return _cache[kind]


def exports(kind, name):
    """True if the `kind` oracle is built and exports `name`"""
    return available(kind) and name in load(kind).orc_exports


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def cpu_info(kind="best"):
    """CPUs this process may use: (threads worth starting, hardware threads, affinity mask size, cgroup quota or 0)"""
    hw = C.c_int(); af = C.c_int(); q = C.c_double()
    eff = load(kind).orc_cpu_info(C.byref(hw), C.byref(af), C.byref(q))
    return eff, hw.value, af.value, q.value


def r128_bench(n_inst, nfram, nblocks, nthreads, steps, warmup=1, pin=True, fsamp=48000.0, kind="best"):
    """the timed CPU baseline (oracle/cpu_bench.inc): persistent pinned workers owning their instances"""
    out = (C.c_double * 6)()
    rc = load(kind).orc_r128_bench(n_inst, nfram, nblocks, nthreads, int(pin), steps, warmup, fsamp, out)
    assert rc == 0
    return {"samples_per_s": out[0], "wall_s": out[1], "threads": int(out[2]), "steps": int(out[3]), "imbalance": out[4], "per_thread": out[5]}


def planar(a):
    """[channels, n] float32 C-contiguous -> (pointer, stride in floats)."""
    assert a.dtype == np.float32 and a.flags.c_contiguous and a.ndim == 2
    return ptr(a), a.shape[1]


# ---------------------------------------------------------------- pythonic wrappers
class Ebu:
    def __init__(self, n_inst, nchan=2, fsamp=48000.0, kind="best"):
        self.L = load(kind)
        self.n, self.nchan = n_inst, nchan
        self.h = self.L.orc_ebu_create(n_inst, nchan, fsamp)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_ebu_destroy(self.h)
            self.h = None

    def integr(self, cmd, inst=-1):
        self.L.orc_ebu_integr(self.h, inst, {"pause": 0, "start": 1, "reset": 2}[cmd])

    def reset(self, inst=-1):
        self.L.orc_ebu_reset(self.h, inst)

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n * self.nchan
        self.L.orc_ebu_process(self.h, p, s, x.shape[1], nthreads)

    def read(self):
        out = np.empty((self.n, 9), np.float32)
        self.L.orc_ebu_read(self.h, ptr(out))
        return out

    def hist(self, inst):
        hm = np.empty(751, np.int32); hs = np.empty(751, np.int32); c = np.empty(4, np.int32)
        self.L.orc_ebu_hist(self.h, inst, ptr(hm), ptr(hs), ptr(c))
        return hm, hs, c

    def coeffs(self):
        o = np.empty(7, np.float32)
        self.L.orc_ebu_coeffs(self.h, ptr(o))
        return o

    def state(self, inst):
        z = np.empty((self.nchan, 4), np.float32); pw = np.empty(64, np.float32)
        fr = np.empty(1, np.float32); c = np.empty(4, np.int32)
        self.L.orc_ebu_state(self.h, inst, ptr(z), ptr(pw), ptr(fr), ptr(c))
        return z, pw, fr[0], c


def _range_walks_end(h):
    """True if both percentile walks of Ebu_r128_hist::calc_range (ebu_r128_proc.cc:143-147) stop by bin 750 for every
    start bin k: `for (i = k, s = 0; s < a; i++) s += h[i]` and `for (j = 750, s = n; s > b; j--) s -= h[j]` in float,
    with n the int sum of h[k:], a = 0.10f * n, b = 0.95f * n.  Vectorised over k; float32 numpy arithmetic rounds as
    the reference's SSE float code does."""
    h = np.asarray(h, np.int64)
    f = h.astype(np.float32)
    ks = np.arange(751)
    n = np.cumsum(h[::-1])[::-1]                       # n[k] = sum h[k:] (exact)
    nf = n.astype(np.float32)
    a = np.float32(0.10) * nf
    b = np.float32(0.95) * nf
    up = np.zeros(751, np.float32)
    for i in range(751):
        up = np.where(ks <= i, up + f[i], up)
    dn = nf.copy()
    for j in range(750, -1, -1):
        dn = np.where(dn > b, dn - f[j], dn)
    return bool(np.all(~(up < a)) and np.all(~(dn > b)))


def hist_calc(hist_m, cnt_m, hist_s, cnt_s, kind="best"):
    """Ebu_r128_hist::calc_integ + calc_range on given counts -> float32[5]: integrated, integ_thr, range_min,
    range_max, range_thr (-200 where the reference leaves a value unset).  The reference's range walks have no
    upper bound, so the counts are checked first: each histogram's bins must sum to its count word, and above
    2^24 points (where float partial sums stop being exact) both walks must provably end by bin 750.
    kind "best" is the reference build when it has this entry, else the port (pinned to the reference's outputs stored
    in tests/golden/ebu_hist_calc.npz by tests/test_oracle_port.py)."""
    if kind == "best":
        kind = "reference" if exports("reference", "orc_ebu_hist_calc") else "port"
    hm = np.ascontiguousarray(hist_m, np.int32); hs = np.ascontiguousarray(hist_s, np.int32)
    assert hm.shape == (751,) and hs.shape == (751,)
    assert (hm >= 0).all() and (hs >= 0).all()
    assert int(hm.astype(np.int64).sum()) == cnt_m and int(hs.astype(np.int64).sum()) == cnt_s, "bins must sum to the count words"
    assert cnt_m < 2 ** 31 and cnt_s < 2 ** 31
    if cnt_s > 2 ** 24:
        assert _range_walks_end(hs), "calc_range would walk past bin 750"
    out = np.empty(5, np.float32)
    load(kind).orc_ebu_hist_calc(ptr(hm), int(cnt_m), ptr(hs), int(cnt_s), ptr(out))
    return out


def r128_cycle(ebu, tp, x, nfram, nblocks, nthreads):
    """x: [2*n_inst, >= nfram*nblocks]; runs nblocks ebur128_run audio cycles on every instance (tp may be None)."""
    p, s = planar(x)
    assert x.shape[1] >= nfram * nblocks
    ebu.L.orc_r128_cycle(ebu.h, tp.h if tp is not None else None, p, s, nfram, nblocks, nthreads)


class TruePeak:
    def __init__(self, n, fsamp=48000.0, kind="best"):
        self.L = load(kind); self.n = n
        self.h = self.L.orc_tp_create(n, fsamp)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_tp_destroy(self.h); self.h = None

    def process(self, x, mode=0, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n
        self.L.orc_tp_process(self.h, p, s, x.shape[1], mode, nthreads)

    def read(self):
        m = np.empty(self.n, np.float32); p = np.empty(self.n, np.float32)
        self.L.orc_tp_read(self.h, ptr(m), ptr(p))
        return m, p

    def peek(self):
        a = [np.empty(self.n, np.float32) for _ in range(4)]; r = np.empty(self.n, np.int32)
        self.L.orc_tp_peek(self.h, *[ptr(v) for v in a], ptr(r))
        return (*a, r)

    def reset(self, inst=-1):
        self.L.orc_tp_reset(self.h, inst)

    def coeffs(self):
        w = np.empty(4, np.float32); t = np.empty(120, np.float32)
        self.L.orc_tp_coeffs(self.h, ptr(w), ptr(t))
        return w, t


def tp_upsample(x, fsamp=48000.0, block=1024, kind="best"):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(4 * x.size, np.float32)
    load(kind).orc_tp_upsample(fsamp, ptr(x), x.size, block, ptr(out))
    return out


class Kmeter:
    def __init__(self, n, fsamp=48000.0, kind="best"):
        self.L = load(kind); self.n = n
        self.h = self.L.orc_km_create(n, fsamp)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_km_destroy(self.h); self.h = None

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n
        self.L.orc_km_process(self.h, p, s, x.shape[1], nthreads)

    def read(self):
        r = np.empty(self.n, np.float32); p = np.empty(self.n, np.float32)
        self.L.orc_km_read(self.h, ptr(r), ptr(p))
        return r, p

    def peek(self):
        s = np.empty((self.n, 8), np.float32)
        self.L.orc_km_peek(self.h, ptr(s))
        return s

    def reset(self, inst=-1):
        self.L.orc_km_reset(self.h, inst)

    def coeffs(self):
        o = np.empty(1, np.float32); h = np.empty(1, np.int32)
        self.L.orc_km_coeffs(self.h, ptr(o), ptr(h))
        return o[0], int(h[0])


PPM_VU, PPM_IEC1, PPM_IEC2, PPM_MS = 0, 1, 2, 3


class Needle:
    """kind 0 VU / 1 IEC-I / 2 IEC-II: n mono meters; kind 3 M/S PPM: n stereo pairs, two meters (M, S) per pair."""

    def __init__(self, n, kind, fsamp=48000.0, oracle="best"):
        self.L = load(oracle); self.n, self.kind = n, kind
        self.nm = 2 * n if kind == PPM_MS else n
        self.h = self.L.orc_ppm_create(n, fsamp, kind)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_ppm_destroy(self.h); self.h = None

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.nm
        self.L.orc_ppm_process(self.h, p, s, x.shape[1], nthreads)

    def read(self):
        o = np.empty(self.nm, np.float32)
        self.L.orc_ppm_read(self.h, ptr(o))
        return o

    def peek(self):
        s = np.empty((self.nm, 4), np.float32)
        self.L.orc_ppm_peek(self.h, ptr(s))
        return s

    def set_gain(self, db_m, db_s):
        self.L.orc_ppm_set_gain(self.h, db_m, db_s)

    def coeffs(self):
        w = np.empty(4, np.float32)
        self.L.orc_ppm_coeffs(self.h, ptr(w))
        return w


class EbuPlugin:
    """the reference's EBUr128 plugin run through its own ebur128_run (reference build only)"""

    def __init__(self, n, rate=48000.0, dbtp=True):
        self.L = load("reference"); self.n = n
        self.h = self.L.orc_ebuplug_create(n, rate, int(dbtp))
        assert self.h

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_ebuplug_destroy(self.h); self.h = None

    def run(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == 2 * self.n
        self.L.orc_ebuplug_run(self.h, p, s, x.shape[1], nthreads)

    def read(self):
        o = np.empty((self.n, 10), np.float32)
        self.L.orc_ebuplug_read(self.h, ptr(o))
        return o


class Bitmeter:
    def __init__(self, n, rate=48000.0, oracle="best"):
        self.L = load(oracle); self.n = n
        self.h = self.L.orc_bim_create(n, rate)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_bim_destroy(self.h); self.h = None

    def mode(self, average, integrating=True):
        self.L.orc_bim_mode(self.h, int(average), int(integrating))

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n
        self.L.orc_bim_process(self.h, p, s, x.shape[1], nthreads)

    def read(self, inst):
        h = np.empty(584, np.int32); c = np.empty(5, np.int32); mm = np.empty(2, np.float32); it = np.empty(1, np.int64)
        self.L.orc_bim_read(self.h, inst, ptr(h), ptr(c), ptr(mm), ptr(it))
        return h, c, mm, int(it[0])


class SigDist:
    def __init__(self, n, rate=48000.0, oracle="best"):
        self.L = load(oracle); self.n = n
        self.h = self.L.orc_sdh_create(n, rate)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_sdh_destroy(self.h); self.h = None

    def integrate(self, on=True):
        self.L.orc_sdh_integrate(self.h, int(on))

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n
        self.L.orc_sdh_process(self.h, p, s, x.shape[1], nthreads)

    def read(self, inst):
        h = np.empty(361, np.int32); mp = np.empty(2, np.int32); av = np.empty(3, np.float64); it = np.empty(1, np.int64)
        self.L.orc_sdh_read(self.h, inst, ptr(h), ptr(mp), ptr(av), ptr(it))
        return h, mp, av, int(it[0])


class Stcorr:
    def __init__(self, n, fsamp=48000, flp=2e3, tcf=0.3, kind="best"):
        self.L = load(kind); self.n = n
        self.h = self.L.orc_cor_create(n, int(fsamp), flp, tcf)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_cor_destroy(self.h); self.h = None

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == 2 * self.n
        self.L.orc_cor_process(self.h, p, s, x.shape[1], nthreads)

    def read(self):
        o = np.empty(self.n, np.float32)
        self.L.orc_cor_read(self.h, ptr(o))
        return o

    def peek(self):
        s = np.empty((self.n, 5), np.float32)
        self.L.orc_cor_peek(self.h, ptr(s))
        return s

    def coeffs(self):
        w = np.empty(2, np.float32)
        self.L.orc_cor_coeffs(self.h, ptr(w))
        return w


class Spectr30:
    def __init__(self, n_inst, nchan=2, rate=48000.0, kind="best"):
        self.L = load(kind); self.n, self.nchan = n_inst, nchan
        self.h = self.L.orc_spec_create(n_inst, nchan, rate)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_spec_destroy(self.h); self.h = None

    def process(self, x, speed=1.0, reset=-4.0, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n * self.nchan
        self.L.orc_spec_process(self.h, p, s, x.shape[1], speed, reset, nthreads)

    def read(self):
        o = np.empty((self.n, 60), np.float32)
        self.L.orc_spec_read(self.h, ptr(o))
        return o

    def state(self, inst):
        z = np.empty((30, 6, 2), np.float64); v = np.empty(30, np.float32); m = np.empty(30, np.float32)
        self.L.orc_spec_state(self.h, inst, ptr(z), ptr(v), ptr(m))
        return z, v, m

    def coeffs(self):
        W = np.empty((30, 6, 6), np.float64)
        self.L.orc_spec_coeffs(self.h, ptr(W))
        return W


class Dr14:
    """dr14_run for n instances; read() -> [n, 12] = v_rms[2] v_peak[2] m_peak[2] m_rms[2] dr[2] dr_total block_count"""

    def __init__(self, n_inst, nch=2, rate=48000.0, dr_mode=True, kind="best"):
        self.L = load(kind); self.n, self.nch = n_inst, nch
        self.h = self.L.orc_dr14_create(n_inst, nch, rate, int(dr_mode))
        assert self.h

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_dr14_destroy(self.h); self.h = None

    def process(self, x, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == self.n * self.nch
        self.L.orc_dr14_process(self.h, p, s, x.shape[1], nthreads)

    def reset(self):
        self.L.orc_dr14_reset(self.h)

    def read(self):
        out = np.empty((self.n, 12), np.float32)
        self.L.orc_dr14_read(self.h, ptr(out))
        return out


class Phasewheel:
    def __init__(self, n_inst, fft_bins=1024, rate=48000.0, kind="port"):
        self.L = load(kind); self.n, self.bins = n_inst, fft_bins
        self.h = self.L.orc_pw_create(n_inst, fft_bins, rate)
        if not self.h:
            raise RuntimeError("phasewheel oracle unavailable in kind=%s (FFTW3 absent)" % kind)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_pw_destroy(self.h); self.h = None

    def set_mode(self, mode):
        """0: phasewheel, 1: stereoscope process_audio (read() then returns lr[] in place of phase[])"""
        self.L.orc_pw_set_mode(self.h, mode)

    def process(self, x, db_thresh=1e-6, nthreads=1):
        p, s = planar(x)
        assert x.shape[0] == 2 * self.n
        return self.L.orc_pw_process(self.h, p, s, x.shape[1], db_thresh, nthreads)

    def read(self):
        ph = np.empty((self.n, self.bins), np.float32); lv = np.empty((self.n, self.bins), np.float32)
        pk = np.empty(self.n, np.float32)
        self.L.orc_pw_read(self.h, ptr(ph), ptr(lv), ptr(pk))
        return ph, lv, pk

    def raw(self, inst):
        a = [np.empty(self.bins, np.float32) for _ in range(4)]
        self.L.orc_pw_raw(self.h, inst, *[ptr(v) for v in a])
        return a
