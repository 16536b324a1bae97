"""Time of b200m_dr14_run_device per block: DR mode, stereo, one shared window phase and, for libraries that have
b200m_dr14_control, 64 staggered phases (every 64th instance reset after each of 64 warm-up blocks).  The libraries given with --lib
are alternated in one session, so that two builds can be compared; the GPU's name and power limit are read at the start and
printed with the results (one JSON line).

    python meters.lv2_b200/host/dr14_run_cost.py [--lib meters.lv2_b200/libb200meters.so ...] [--instances 8192] [--nframes 1024]
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


def _load(path):
    L = C.CDLL(os.path.abspath(path))
    L.b200m_dr14_create.argtypes = [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_double, C.c_int]
    L.b200m_dr14_run_device.argtypes = [_v, _v, C.c_size_t, C.c_uint32, _v]
    L.b200m_dr14_destroy.argtypes = [_v]
    if hasattr(L, "b200m_dr14_control"):
        L.b200m_dr14_control.argtypes = [_v, _v, C.c_uint32, C.c_int, _v]
    return L


def _time(L, x, n_inst, nframes, stagger, iters):
    st = _v(torch.cuda.current_stream().cuda_stream)
    h = _v()
    assert L.b200m_dr14_create(C.byref(h), 0, n_inst, 2, 48000.0, 1) == 0
    run = lambda: L.b200m_dr14_run_device(h, _v(x.data_ptr()), nframes, nframes, st)
    if stagger:
        for k in range(64):
            assert run() == 0
            sel = np.arange(k, n_inst, 64, dtype=np.uint32)
            assert L.b200m_dr14_control(h, _v(sel.ctypes.data), sel.size, 1, st) == 0
    for _ in range(50):
        assert run() == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    L.b200m_dr14_destroy(h)
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
    for _ in range(a.runs):
        for p, L in libs.items():
            res.setdefault(p + " shared phase", []).append(round(_time(L, x, a.instances, a.nframes, False, a.iters), 2))
            if hasattr(L, "b200m_dr14_control"):
                res.setdefault(p + " 64 phases", []).append(round(_time(L, x, a.instances, a.nframes, True, a.iters), 2))
    print(json.dumps({"gpu": gpu, "stereo_instances": a.instances, "nframes": a.nframes, "us_per_block": res}))


if __name__ == "__main__":
    main()
