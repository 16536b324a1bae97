"""Time per block of stereo banks with one shared phase against 64 staggered phases, 48 kHz, 8192 instances x 1024 frames:
  r128  b200m_r128_run_device, dBTP on, in tolerance mode (the fused K-weighting + true-peak kernel) and in exact mode; the
        64 phases of its 50 ms fragment clock, for libraries that have B200M_R128_NEW, come from every 64th instance getting
        B200M_R128_NEW after each of 64 warm-up blocks;
  dr14  b200m_dr14_run_device, DR mode; the 64 phases of its 3 s window clock, for libraries that have b200m_dr14_control, come
        from every 64th instance being reset after each of 64 warm-up blocks.
CUDA events over --iters blocks after 50 warm-up blocks.  The libraries given with --lib are alternated in one session, their
order reversed on every other run, so that two builds can be compared.  The GPU's name and power limit are read at the start and
printed with the results (one JSON line).

    python meters.lv2_b200/host/phase_cost.py [--banks r128,dr14] [--lib meters.lv2_b200/libb200meters.so ...] [--instances 8192]
                                              [--nframes 1024] [--iters 300] [--runs 3]
"""
import ctypes as C
import json

import numpy as np

import _cost
from _cost import B

_v = C.c_void_p
PREC = {"tolerance": B.PREC_FMA, "exact": B.PREC_EXACT}


def _r128(L, x, n_inst, nframes, mode, stagger, iters):
    """us per block, or None when the library has no per-instance fragment clock"""
    st = B._stream_ptr(None)
    h = _v()
    B._ck(L.b200m_r128_create(C.byref(h), 0, n_inst, 48000.0, 1))
    B._ck(L.b200m_r128_set_precision(h, PREC[mode]))
    B._ck(L.b200m_r128_control(h, -1, B.EBUr128.START, st))
    run = lambda: L.b200m_r128_run_device(h, _v(x.data_ptr()), nframes, nframes, st)
    if stagger:
        for k in range(64):
            B._ck(run())
            for i in range(k, n_inst, 64):
                if L.b200m_r128_control(h, i, B.EBUr128.NEW, st) != 0:
                    L.b200m_r128_destroy(h)
                    return None
            B._ck(L.b200m_r128_control(h, -1, B.EBUr128.START, st))
    t = _cost.events(run, iters, 50)
    L.b200m_r128_destroy(h)
    return t


def _dr14(L, x, n_inst, nframes, stagger, iters):
    st = B._stream_ptr(None)
    h = _v()
    B._ck(L.b200m_dr14_create(C.byref(h), 0, n_inst, 2, 48000.0, 1))
    run = lambda: L.b200m_dr14_run_device(h, _v(x.data_ptr()), nframes, nframes, st)
    if stagger:
        for k in range(64):
            B._ck(run())
            sel = np.arange(k, n_inst, 64, dtype=np.uint32)
            B._ck(L.b200m_dr14_control(h, _v(sel.ctypes.data), sel.size, 1, st))
    t = _cost.events(run, iters, 50)
    L.b200m_dr14_destroy(h)
    return t


def r128(p, L, x, a, res):
    for mode in PREC:
        res.setdefault(f"{p} {mode} one phase", []).append(_r128(L, x, a.instances, a.nframes, mode, False, a.iters))
        t = _r128(L, x, a.instances, a.nframes, mode, True, a.iters)
        if t is not None:
            res.setdefault(f"{p} {mode} 64 phases", []).append(t)


def dr14(p, L, x, a, res):
    res.setdefault(p + " shared phase", []).append(_dr14(L, x, a.instances, a.nframes, False, a.iters))
    if hasattr(L, "b200m_dr14_control"):
        res.setdefault(p + " 64 phases", []).append(_dr14(L, x, a.instances, a.nframes, True, a.iters))


BANKS = {"r128": r128, "dr14": dr14}


def main():
    a = _cost.parser(__doc__, banks=BANKS, lib=True, instances=8192, nframes=1024, iters=300, runs=3).parse_args()
    libs = {p: B.load_lib(p) for p in (a.lib or [B.LIB_PATH])}
    out = {"gpu": _cost.gpu()}
    for name in a.banks.split(","):
        x = _cost.noise(2 * a.instances, a.nframes)
        res = {}
        for r in range(a.runs):
            for p in _cost.alternate(libs, r):
                BANKS[name](p, libs[p], x, a, res)
        out[name] = {"stereo_instances": a.instances, "nframes": a.nframes, "us_per_block": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
