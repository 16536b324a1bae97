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
import argparse
import ctypes as C
import json
import os
import subprocess

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
_v = C.c_void_p
R128_START = 1
PREC = {"tolerance": 1, "exact": 0}


def _load(path):
    L = C.CDLL(os.path.abspath(path))
    L.b200m_r128_create.argtypes = [C.POINTER(_v), C.c_int, C.c_uint32, C.c_float, C.c_int]
    if hasattr(L, "b200m_r128_create_nch"):
        L.b200m_r128_create_nch.argtypes = [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_float, C.c_int]
    if hasattr(L, "b200m_r128_create_weighted"):
        L.b200m_r128_create_weighted.argtypes = [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, _v, C.c_float, C.c_int]
    L.b200m_r128_run_device.argtypes = [_v, _v, C.c_size_t, C.c_uint32, _v]
    L.b200m_r128_control.argtypes = [_v, C.c_int32, C.c_int, _v]
    L.b200m_r128_set_precision.argtypes = [_v, C.c_int]
    L.b200m_r128_destroy.argtypes = [_v]
    return L


def _time(L, x, nchan, nframes, mode, iters, weighted=False):
    """us per block, or None when the library has no b200m_r128_create_nch and nchan != 2 (weighted: no b200m_r128_create_weighted)"""
    st = _v(torch.cuda.current_stream().cuda_stream)
    h = _v()
    n_inst = x.shape[0] // nchan
    if weighted:
        if not hasattr(L, "b200m_r128_create_weighted"):
            return None
        g = (C.c_float * nchan)(*[1.41 if c % 8 in (3, 4) else 1.0 for c in range(nchan)])
        assert L.b200m_r128_create_weighted(C.byref(h), 0, n_inst, nchan, C.cast(g, _v), 48000.0, 1) == 0
    elif hasattr(L, "b200m_r128_create_nch"):
        assert L.b200m_r128_create_nch(C.byref(h), 0, n_inst, nchan, 48000.0, 1) == 0
    elif nchan == 2:
        assert L.b200m_r128_create(C.byref(h), 0, n_inst, 48000.0, 1) == 0
    else:
        return None
    assert L.b200m_r128_set_precision(h, PREC[mode]) == 0
    assert L.b200m_r128_control(h, -1, R128_START, st) == 0
    run = lambda: L.b200m_r128_run_device(h, _v(x.data_ptr()), nframes, nframes, st)
    for _ in range(50):
        assert run() == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    L.b200m_r128_destroy(h)
    return a.elapsed_time(b) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--channels", type=int, default=16380)
    ap.add_argument("--nframes", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--weighted", default="7,11,22,32", help="channels per instance of the weighted layouts ('' for none)")
    a = ap.parse_args()
    libs = {p: _load(p) for p in (a.lib or [os.path.join(HERE, "..", "libb200meters.so")])}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    x = (torch.rand(a.channels, a.nframes, device="cuda") * 2 - 1) * 0.5
    res = {}
    for r in range(a.runs):
        for p, L in (list(libs.items()) if r % 2 == 0 else list(libs.items())[::-1]):
            for mode in PREC:
                for nchan in range(1, 6):
                    if a.channels % nchan:
                        continue
                    t = _time(L, x, nchan, a.nframes, mode, a.iters)
                    if t is not None:
                        res.setdefault(f"{p} {mode} nchan={nchan}", []).append(round(t, 2))
                for nchan in [int(v) for v in a.weighted.split(",") if v]:
                    t = _time(L, x, nchan, a.nframes, mode, a.iters, weighted=True)
                    if t is not None:
                        res.setdefault(f"{p} {mode} weighted nchan={nchan} x {a.channels // nchan}", []).append(round(t, 2))
    print(json.dumps({"gpu": gpu, "channels": a.channels, "nframes": a.nframes, "us_per_block": res}))


if __name__ == "__main__":
    main()
