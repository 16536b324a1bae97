"""Cost of ragged blocks in the true-peak / K-meter, needle-meter, correlation and spectrum banks (b200m_*_process_ragged_device),
48 kHz, 1024-frame blocks:
  tpk   16384 channels, true peak + K-meter, process()
  vu    16384 VU meters          iec2  16384 IEC type II meters
  cor   8192 pairs, exact        cor_scan  8192 pairs, B200M_PREC_FMA
  spec  4096 stereo instances, exact                spec_fma  the same in B200M_PREC_FMA
Four forms per bank: the plain call, a ragged call with every length equal to nfram (the same call), and blocks in which 1 % / 50 %
of the rows end early (a random length below nfram).  Each figure is the CUDA-event time per block over --iters blocks, next to the
host's wall time per call in the same loop (the C entry points are called directly, with their arguments prepared beforehand).
Every figure is taken --runs times, the forms alternating.  The GPU's name and power limit are read in the same call and printed
with the results (one JSON line).

    python meters.lv2_b200/host/meters_ragged_cost.py [--nframes 1024] [--iters 300] [--runs 3] [--banks tpk,vu,...]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import meters_lv2_b200 as B  # noqa: E402


def _time(fn, iters):
    for _ in range(20):
        B._ck(fn())
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    host = time.perf_counter() - t0
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) / iters * 1e3, 2), round(host / iters * 1e6, 2)


def _forms(n, nf, rng):
    full = np.full(n, nf, np.uint32)
    forms = {"plain": None, "ragged all nfram": full}
    for pct in (1, 50):
        lens = full.copy()
        idx = rng.choice(n, size=max(1, n * pct // 100), replace=False)
        lens[idx] = rng.integers(0, nf, size=idx.size)
        forms[f"{pct}% end early"] = lens
    return forms


# bank name -> (units, rows per unit, constructor, C entry point prefix).  The C ABI is called directly with arguments prepared
# outside the timed loop, so that the figures are the library's, not the Python wrappers'.
BANKS = {
    "tpk": (16384, 1, lambda n: B.TruePeakKmeter(n), "tpk"),
    "vu": (16384, 1, lambda n: B.NeedleMeters(n, B.PPM_VU), "ppm"),
    "iec2": (16384, 1, lambda n: B.NeedleMeters(n, B.PPM_IEC2), "ppm"),
    "cor": (8192, 2, lambda n: B.Stcorrdsp(n), "cor"),
    "cor_scan": (8192, 2, lambda n: _prec(B.Stcorrdsp(n)), "cor"),
    "spec": (4096, 2, lambda n: B.Spectr30(n, 2), "spec"),
    "spec_fma": (4096, 2, lambda n: _prec(B.Spectr30(n, 2)), "spec"),
}


def _call(g, pfx, x, lens, ctl):
    """a closure for one block: the plain device-path call (lens None) or the ragged one"""
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
    plain, rag = getattr(L, "b200m_%s_process_device" % pfx), getattr(L, "b200m_%s_process_ragged_device" % pfx)
    return (lambda: plain(g.h, p, s, nf, st)) if ln is None else (lambda: rag(g.h, p, s, nf, ln, st))


def _prec(g):
    g.set_precision(B.PREC_FMA)
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--nframes", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--banks", default=",".join(BANKS))
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    nf = a.nframes
    out = {"gpu": gpu, "nframes": nf, "us_per_block": {}, "host_us_per_call": {}}
    for name in a.banks.split(","):
        n, per, make, pfx = BANKS[name]
        x = (torch.rand(per * n, nf, device="cuda") * 2 - 1) * 0.5
        ctl = np.tile(np.array([[1.0, -4.0]], np.float32), (n, 1))
        forms = _forms(n, nf, np.random.default_rng(0))
        res, host = {}, {}
        for r in range(a.runs):
            for k in (list(forms) if r % 2 == 0 else list(forms)[::-1]):
                g = make(n)
                dev, hst = _time(_call(g, pfx, x, forms[k], ctl), a.iters)
                res.setdefault(k, []).append(dev)
                host.setdefault(k, []).append(hst)
                g.close()
        out["us_per_block"][f"{name} x{n}"] = res
        out["host_us_per_call"][f"{name} x{n}"] = host
    print(json.dumps(out))


if __name__ == "__main__":
    main()
