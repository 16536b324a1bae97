"""Cost of album DR (b200m_dr14_group_reduce / b200m_dr14_group_finish) for a bank of stereo DR-14 instances whose histograms hold
--seconds of noise at a level drawn per instance and block (about -60 .. 0 dBFS):
  (a) one reduce call (the zeroing of the G output rows, the reduce kernel and the peaks kernel): CUDA events over --iters
      back-to-back calls, and the achieved rate over the histogram read, n_inst x 2 x 8000 x 4 bytes.  G = 1, 64, 1024, 8192
      (album of instance i: i * G // n_inst) and a skewed assignment (one album of half the bank, one album per instance for the
      other half);
  (b) one reduce + finish call (the finish copies G results to the host and synchronises): a host clock over --iters calls.
Both entry points are called through ctypes with prepared arguments.  Each figure is taken --runs times; every album layout's rows
are checked against the G = 1 row (they must sum to it).  The GPU's name and power limit are read in the same call and printed
with the results (one JSON line).

    python meters.lv2_b200/host/dr14_group_cost.py [--instances 8192] [--seconds 60] [--iters 50] [--runs 3]
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


def _events(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) / iters * 1e3, 2)


def _host_clock(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return round((time.perf_counter() - t0) / iters * 1e6, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    n, nch = a.instances, 2
    L = B.lib()
    bank = B.DR14(n, nch, 48000.0, True)
    gen = torch.Generator(device="cuda"); gen.manual_seed(0)
    for _ in range(int(a.seconds * 48000) // 8192):
        lvl = 10.0 ** (torch.rand(n, 1, device="cuda", generator=gen) * -3.0)
        x = (torch.rand(nch * n, 8192, device="cuda", generator=gen) * 2 - 1) * lvl.repeat_interleave(nch, 0)
        bank.run(x)
    torch.cuda.synchronize()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    words = B.dr14_group_words(nch)
    layouts = {f"G={g}": (np.arange(n) * g // n, g) for g in (1, 64, 1024, 8192)}
    half = n // 2
    layouts["skewed"] = (np.concatenate([np.zeros(half, np.int64), 1 + np.arange(n - half)]), 1 + n - half)
    prepared, total = {}, None
    for name, (groups, g) in layouts.items():
        g32 = np.ascontiguousarray(groups.astype(np.uint32))
        d = torch.empty((g, words), dtype=torch.int32, device="cuda")
        p = torch.empty((g, nch, 3), dtype=torch.float32, device="cuda")
        o = np.empty(g, B.DR14_ALBUM_DTYPE)
        bank.group_reduce(groups, d, p)
        s = d.sum(0, dtype=torch.int64)
        total = s if total is None else total
        assert torch.equal(s, total), name                                  # every instance is in one album
        prepared[name] = (g32, g, d, p, o)
    rows = prepared["G=8192"][2] if n == 8192 else None
    nonzero = None if rows is None else round(float((rows[:, :-2] != 0).sum().item()) / n, 1)
    read_mb = n * nch * 8000 * 4 / 1e6

    def reduce_fn(name):
        g32, g, d, p, _ = prepared[name]
        gp, dp, pp = B._np_ptr(g32), C.c_void_p(d.data_ptr()), C.c_void_p(p.data_ptr())
        return lambda: B._ck(L.b200m_dr14_group_reduce(bank.h, gp, g, dp, pp, st))

    def reduce_finish_fn(name):
        g32, g, d, p, o = prepared[name]
        gp, dp, pp, op = B._np_ptr(g32), C.c_void_p(d.data_ptr()), C.c_void_p(p.data_ptr()), B._np_ptr(o)

        def f():
            B._ck(L.b200m_dr14_group_reduce(bank.h, gp, g, dp, pp, st))
            B._ck(L.b200m_dr14_group_finish(bank.h, dp, pp, 1, g, op, st))
        return f

    red, both = {}, {}
    names = list(prepared)
    for r in range(a.runs):
        for name in (names if r % 2 == 0 else names[::-1]):
            red.setdefault(name, []).append(_events(reduce_fn(name), a.iters))
            both.setdefault(name, []).append(_host_clock(reduce_finish_fn(name), a.iters))
    gbs = {k: [round(read_mb / t * 1e3, 1) for t in v] for k, v in red.items()}              # MB / us = TB/s
    print(json.dumps({"gpu": gpu, "stereo_instances": n, "seconds": a.seconds, "hist_read_MB": round(read_mb, 1),
                      "nonzero_words_per_instance": nonzero, "reduce_us": red, "reduce_GBps": gbs, "reduce_finish_us": both}))


if __name__ == "__main__":
    main()
