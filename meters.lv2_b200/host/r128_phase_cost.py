"""Time of b200m_r128_run_device per block: stereo, dBTP on, in tolerance mode (the fused K-weighting + true-peak kernel) and in
exact mode, with one shared fragment phase and, for libraries that have B200M_R128_NEW, 64 staggered phases (every 64th instance
gets B200M_R128_NEW after each of 64 warm-up blocks).  The libraries given with --lib are alternated in one session, so that two
builds can be compared (their order is reversed on every other run); the GPU's name and power limit are read at the start and printed with the results (one JSON line).

    python meters.lv2_b200/host/r128_phase_cost.py [--lib meters.lv2_b200/libb200meters.so ...] [--instances 8192] [--nframes 1024]
"""
import argparse
import ctypes as C
import json
import os
import subprocess

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
_v = C.c_void_p
R128_START, R128_NEW = 1, 6
PREC = {"tolerance": 1, "exact": 0}


def _load(path):
    L = C.CDLL(os.path.abspath(path))
    L.b200m_r128_create.argtypes = [C.POINTER(_v), C.c_int, C.c_uint32, C.c_float, C.c_int]
    L.b200m_r128_run_device.argtypes = [_v, _v, C.c_size_t, C.c_uint32, _v]
    L.b200m_r128_control.argtypes = [_v, C.c_int32, C.c_int, _v]
    L.b200m_r128_set_precision.argtypes = [_v, C.c_int]
    L.b200m_r128_destroy.argtypes = [_v]
    return L


def _time(L, x, n_inst, nframes, mode, stagger, iters):
    """us per block, or None when the library has no per-instance fragment clock"""
    st = _v(torch.cuda.current_stream().cuda_stream)
    h = _v()
    assert L.b200m_r128_create(C.byref(h), 0, n_inst, 48000.0, 1) == 0
    assert L.b200m_r128_set_precision(h, PREC[mode]) == 0
    assert L.b200m_r128_control(h, -1, R128_START, st) == 0
    run = lambda: L.b200m_r128_run_device(h, _v(x.data_ptr()), nframes, nframes, st)
    if stagger:
        for k in range(64):
            assert run() == 0
            for i in range(k, n_inst, 64):
                if L.b200m_r128_control(h, i, R128_NEW, st) != 0:
                    L.b200m_r128_destroy(h)
                    return None
            assert L.b200m_r128_control(h, -1, R128_START, st) == 0
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
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--nframes", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=300)
    a = ap.parse_args()
    libs = {p: _load(p) for p in (a.lib or [os.path.join(HERE, "..", "libb200meters.so")])}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    x = (torch.rand(2 * a.instances, a.nframes, device="cuda") * 2 - 1) * 0.5
    res = {}
    for r in range(a.runs):
        for p, L in (list(libs.items()) if r % 2 == 0 else list(libs.items())[::-1]):
            for mode in PREC:
                res.setdefault(f"{p} {mode} one phase", []).append(round(_time(L, x, a.instances, a.nframes, mode, False, a.iters), 2))
                t = _time(L, x, a.instances, a.nframes, mode, True, a.iters)
                if t is not None:
                    res.setdefault(f"{p} {mode} 64 phases", []).append(round(t, 2))
    print(json.dumps({"gpu": gpu, "stereo_instances": a.instances, "nframes": a.nframes, "us_per_block": res}))


if __name__ == "__main__":
    main()
