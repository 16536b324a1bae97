"""Cost of ragged blocks (b200m_*_process_ragged_device / b200m_*_run_ragged_device), 48 kHz, 1024-frame blocks:
  tpk       16384 channels, true peak + K-meter, process()
  vu        16384 VU meters                  iec2      16384 IEC type II meters
  cor       8192 pairs, exact                cor_scan  8192 pairs, B200M_PREC_FMA
  spec      4096 stereo instances, exact     spec_fma  the same in B200M_PREC_FMA
  bim       16384 bit-meter instances (integrating)
  sdh       16384 SigDistHist instances (integrating)
  pw        2048 phasewheel instances, fft_bins 1024
  pw_cor    the same with an attached correlation bank of 2048 pairs
  dr14      8192 stereo DR-14 instances, DR mode, through DR14.run
Four forms per bank: the plain call, a ragged call with every length equal to nfram (the same call), and blocks in which 1 % / 50 %
of the rows end early (a random length below nfram).  Each figure is the CUDA-event time per block over --iters blocks, next to the
host's wall time per call in the same loop.  Every bank but dr14 is timed through its C entry points, with their arguments
prepared beforehand; dr14's host time is that of DR14.run (the enqueue, the lengths' upload and the phase mirror; the host runs
ahead of the device until the launch queue is full, so where the two agree the host may be the bound).  A bank is fresh for every
figure, so a phasewheel's first ending-early block moves its instances' clocks apart and the rest of the loop runs the
per-instance form.  Every figure is taken --runs times, the forms alternating.  The GPU's name and power limit are read in the
same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/ragged_cost.py [--banks tpk,vu,...] [--instances N] [--nframes 1024] [--iters 300] [--runs 3]
"""
import ctypes as C
import json

import numpy as np

import _cost
from _cost import B


def _prec(g):
    g.set_precision(B.PREC_FMA)
    return g


def _sdh(n):
    g = B.SigDistHist(n)
    g.control(B.CTL_START)
    return g


def _pw_cor(n):
    g = B.Phasewheel(n, 1024)
    g._c = B.Stcorrdsp(n)
    g.attach_cor(g._c)
    return g


# bank -> (units, rows per unit, constructor, C entry point prefix or None for DR14.run)
BANKS = {
    "tpk": (16384, 1, lambda n: B.TruePeakKmeter(n), "tpk"),
    "vu": (16384, 1, lambda n: B.NeedleMeters(n, B.PPM_VU), "ppm"),
    "iec2": (16384, 1, lambda n: B.NeedleMeters(n, B.PPM_IEC2), "ppm"),
    "cor": (8192, 2, lambda n: B.Stcorrdsp(n), "cor"),
    "cor_scan": (8192, 2, lambda n: _prec(B.Stcorrdsp(n)), "cor"),
    "spec": (4096, 2, lambda n: B.Spectr30(n, 2), "spec"),
    "spec_fma": (4096, 2, lambda n: _prec(B.Spectr30(n, 2)), "spec"),
    "bim": (16384, 1, lambda n: B.Bitmeter(n), "bim"),
    "sdh": (16384, 1, _sdh, "sdh"),
    "pw": (2048, 2, lambda n: B.Phasewheel(n, 1024), "pw"),
    "pw_cor": (2048, 2, _pw_cor, "pw"),
    "dr14": (8192, 2, lambda n: B.DR14(n, 2, 48000.0, True), None),
}


def _call(g, pfx, x, lens, ctl):
    """a closure for one block: the plain device-path call (lens None) or the ragged one; ctl: the spectrum's per-instance
    controls"""
    if pfx is None:
        return lambda: g.run(x, lengths=lens)
    L = B.lib()
    p, s, _, nf = B._dev_ptr(x)
    st = B._stream_ptr(None)
    ln = None if lens is None else B._np_ptr(lens)
    if pfx == "tpk":
        return (lambda: L.b200m_tpk_process_device(g.h, p, s, nf, B.TP_MODE_PROCESS, st)) if ln is None else \
               (lambda: L.b200m_tpk_process_ragged_device(g.h, p, s, nf, ln, st))
    if pfx == "spec":
        c = B._np_ptr(ctl)
        return (lambda: L.b200m_spec_process_ctl_device(g.h, p, s, nf, c, st)) if ln is None else \
               (lambda: L.b200m_spec_process_ragged_device(g.h, p, s, nf, c, ln, st))
    if pfx == "pw":
        fired = C.c_int(0)
        return (lambda: L.b200m_pw_process_device(g.h, p, s, nf, 1e-6, C.byref(fired), st)) if ln is None else \
               (lambda: L.b200m_pw_process_ragged_device(g.h, p, s, nf, ln, 1e-6, C.byref(fired), st))
    verb = "run" if pfx in ("bim", "sdh") else "process"
    plain, rag = getattr(L, f"b200m_{pfx}_{verb}_device"), getattr(L, f"b200m_{pfx}_{verb}_ragged_device")
    return (lambda: plain(g.h, p, s, nf, st)) if ln is None else (lambda: rag(g.h, p, s, nf, ln, st))


def main():
    a = _cost.parser(__doc__, banks=BANKS, instances=None, nframes=1024, iters=300, runs=3).parse_args()
    nf = a.nframes
    out = {"gpu": _cost.gpu(), "nframes": nf, "us_per_block": {}, "host_us_per_call": {}}
    for name in a.banks.split(","):
        n, per, make, pfx = BANKS[name]
        n = a.instances or n
        x = _cost.noise(per * n, nf)
        forms = _cost.ragged_forms(n, nf, np.random.default_rng(0), ab=name == "dr14")
        ctl = np.tile(np.array([[1.0, -4.0]], np.float32), (n, 1))
        res, host = {}, {}
        for r in range(a.runs):
            for k in _cost.alternate(forms, r):
                g = make(n)
                dev, hst = _cost.events(_call(g, pfx, x, forms[k], ctl), a.iters, 20, host=True)
                res.setdefault(k, []).append(dev)
                host.setdefault(k, []).append(hst)
                g.close()
                if hasattr(g, "_c"):
                    g._c.close()
        out["us_per_block"][f"{name} x{n}"] = res
        out["host_us_per_call"][f"{name} x{n}"] = host
    print(json.dumps(out))


if __name__ == "__main__":
    main()
