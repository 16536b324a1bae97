"""Time of b200m_r128_run_device per block for instances of 1..5 channels: 16380 channels (divisible by 1..5) x 1024 frames, dBTP on,
in tolerance mode (the fused K-weighting + true-peak kernel: 128-channel slabs for 1, 2, 4 channels, 120-channel slabs for 3, 5) and
in exact mode (K-weighting + tpmax_kernel, and for 3 and 5 channels r128_hold_kernel).  CUDA events over --iters blocks after 50
warm-up blocks; --runs runs, the libraries given with --lib alternated (order reversed on every other run).  A library without
b200m_r128_create_nch is timed at 2 channels only.  The GPU's name and power limit are read at the start and printed with the
results (one JSON line).
Weighted layouts (b200m_r128_create_weighted, --weighted, default 7, 11, 22 and 32 channels per instance) are timed in the same
session, in both modes, as floor (channels / nchan) instances with BS.1770-4-style weights (1.41 on two of every eight channels):
these banks run the run-time channel-count K-weighting kernel and, in tolerance mode, the tensor-core FIR behind it (they have no
fused form).  A library without b200m_r128_create_weighted skips them.

    python meters.lv2_b200/host/r128_nch_cost.py [--lib meters.lv2_b200/libb200meters.so ...] [--channels 16380] [--nframes 1024]
                                                 [--weighted 7,11,22,32]
"""
import ctypes as C
import json

import _cost
from _cost import B

_v = C.c_void_p
PREC = {"tolerance": B.PREC_FMA, "exact": B.PREC_EXACT}


def _time(L, x, nchan, nframes, mode, iters, weighted=False):
    """us per block, or None when the library has no b200m_r128_create_nch and nchan != 2 (weighted: no b200m_r128_create_weighted)"""
    st = B._stream_ptr(None)
    h = _v()
    n_inst = x.shape[0] // nchan
    if weighted:
        if not hasattr(L, "b200m_r128_create_weighted"):
            return None
        g = (C.c_float * nchan)(*[1.41 if c % 8 in (3, 4) else 1.0 for c in range(nchan)])
        B._ck(L.b200m_r128_create_weighted(C.byref(h), 0, n_inst, nchan, C.cast(g, _v), 48000.0, 1))
    elif hasattr(L, "b200m_r128_create_nch"):
        B._ck(L.b200m_r128_create_nch(C.byref(h), 0, n_inst, nchan, 48000.0, 1))
    elif nchan == 2:
        B._ck(L.b200m_r128_create(C.byref(h), 0, n_inst, 48000.0, 1))
    else:
        return None
    B._ck(L.b200m_r128_set_precision(h, PREC[mode]))
    B._ck(L.b200m_r128_control(h, -1, B.EBUr128.START, st))
    t = _cost.events(lambda: L.b200m_r128_run_device(h, _v(x.data_ptr()), nframes, nframes, st), iters, 50)
    L.b200m_r128_destroy(h)
    return t


def main():
    ap = _cost.parser(__doc__, lib=True, nframes=1024, iters=300, runs=3)
    ap.add_argument("--channels", type=int, default=16380)
    ap.add_argument("--weighted", default="7,11,22,32", help="channels per instance of the weighted layouts ('' for none)")
    a = ap.parse_args()
    libs = {p: B.load_lib(p) for p in (a.lib or [B.LIB_PATH])}
    gpu = _cost.gpu()
    x = _cost.noise(a.channels, a.nframes)
    res = {}
    for r in range(a.runs):
        for p in _cost.alternate(libs, r):
            L = libs[p]
            for mode in PREC:
                for nchan in range(1, 6):
                    if a.channels % nchan:
                        continue
                    t = _time(L, x, nchan, a.nframes, mode, a.iters)
                    if t is not None:
                        res.setdefault(f"{p} {mode} nchan={nchan}", []).append(t)
                for nchan in [int(v) for v in a.weighted.split(",") if v]:
                    t = _time(L, x, nchan, a.nframes, mode, a.iters, weighted=True)
                    if t is not None:
                        res.setdefault(f"{p} {mode} weighted nchan={nchan} x {a.channels // nchan}", []).append(t)
    print(json.dumps({"gpu": gpu, "channels": a.channels, "nframes": a.nframes, "us_per_block": res}))


if __name__ == "__main__":
    main()
