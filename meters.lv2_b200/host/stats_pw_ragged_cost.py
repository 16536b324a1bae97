"""Cost of ragged blocks in the bit-meter, SigDistHist and phasewheel banks (b200m_bim_run_ragged_device,
b200m_sdh_run_ragged_device, b200m_pw_process_ragged_device), 48 kHz, 1024-frame blocks:
  bim      16384 bit-meter instances (integrating)
  sdh      16384 SigDistHist instances (integrating)
  pw       2048 phasewheel instances, fft_bins 1024
  pw_cor   the same with an attached correlation bank of 2048 pairs
Four forms per bank: the plain call, a ragged call with every length equal to nfram (the same call), and blocks in which 1 % / 50 %
of the instances end early (a random length below nfram).  Each figure is the CUDA-event time per block over --iters blocks, next to
the host's wall time per call in the same loop (the C entry points are called directly, with their arguments prepared beforehand).
A phasewheel bank is fresh for every figure, so its first ending-early block moves its instances' clocks apart and the rest of the
loop runs the per-instance form.  Every figure is taken --runs times, the forms alternating.  The GPU's name and power limit are read
in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/stats_pw_ragged_cost.py [--nframes 1024] [--iters 300] [--runs 3] [--banks bim,sdh,pw,pw_cor]
"""
import argparse
import ctypes as C
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


def _make(name, n):
    if name == "bim":
        return B.Bitmeter(n)
    if name == "sdh":
        g = B.SigDistHist(n)
        g.control(B.CTL_START)
        return g
    g = B.Phasewheel(n, 1024)
    if name == "pw_cor":
        g._c = B.Stcorrdsp(n)
        g.attach_cor(g._c)
    return g


# bank name -> (instances, rows per instance)
BANKS = {"bim": (16384, 1), "sdh": (16384, 1), "pw": (2048, 2), "pw_cor": (2048, 2)}


def _call(name, g, x, lens):
    """a closure for one block: the plain device-path call (lens None) or the ragged one"""
    L = B.lib()
    p, s, _, nf = B._dev_ptr(x)
    st = B._stream_ptr(None)
    ln = None if lens is None else B._np_ptr(lens)
    if name in ("bim", "sdh"):
        plain, rag = getattr(L, "b200m_%s_run_device" % name), getattr(L, "b200m_%s_run_ragged_device" % name)
        return (lambda: plain(g.h, p, s, nf, st)) if ln is None else (lambda: rag(g.h, p, s, nf, ln, st))
    fired = C.c_int(0)
    if ln is None:
        return lambda: L.b200m_pw_process_device(g.h, p, s, nf, 1e-6, C.byref(fired), st)
    return lambda: L.b200m_pw_process_ragged_device(g.h, p, s, nf, ln, 1e-6, C.byref(fired), st)


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
        n, per = BANKS[name]
        x = (torch.rand(per * n, nf, device="cuda") * 2 - 1) * 0.5
        forms = _forms(n, nf, np.random.default_rng(0))
        res, host = {}, {}
        for r in range(a.runs):
            for k in (list(forms) if r % 2 == 0 else list(forms)[::-1]):
                g = _make(name, n)
                dev, hst = _time(_call(name, g, x, forms[k]), a.iters)
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
