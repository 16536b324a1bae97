"""Cost of the DR-14 bank's window log (b200m_dr14_log_enable), stereo, DR mode, device path:
  (a) b200m_dr14_run_device per 1024-frame block with the log off and on (capacity 16 points = 48 s), the two alternating, each
      timed over --iters blocks: 3 s windows and more of audio, so that the blocks in which windows close (and the log writes its
      points) are in the window;
  (b) one b200m_dr14_log_drain of every instance's full log (8192 x 16 points): the drain kernel and the device-to-host copy into
      pageable memory, as DR14.log_drain does it.
(a) is a CUDA-event time per block over --iters blocks, (b) a host clock around the synchronous drain; every figure is taken --runs
times.  The GPU's name and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/dr14_log_cost.py [--instances 8192] [--nframes 1024] [--iters 600] [--runs 3] [--capacity 16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import meters_lv2_b200 as B  # noqa: E402

RATE = 48000.0
WINDOW = 144001                 # rintf (3 * 48000) + 1 frames


def _events(fn, iters):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) / iters * 1e3, 2)


def _run(x, n, log, cap, iters):
    bk = B.DR14(n, 2, RATE, True)
    if log:
        bk.log_enable(cap)
    t = _events(lambda: bk.run(x), iters)
    bk.close()
    return t


def _drain(x, n, cap):
    """ms of one drain of a full log: cap points of every instance (written by cap windows of input)"""
    bk = B.DR14(n, 2, RATE, True)
    bk.log_enable(cap)
    for _ in range(-(-cap * WINDOW // x.shape[1])):
        bk.run(x)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, cnt, _ = bk.log_drain()
    t = (time.perf_counter() - t0) * 1e3
    assert (cnt == cap).all()
    bk.close()
    return round(t, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--nframes", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=600)
    ap.add_argument("--capacity", type=int, default=16)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    n, nf = a.instances, a.nframes
    x = (torch.rand(2 * n, nf, device="cuda") * 2 - 1) * 0.5
    res = {}
    for r in range(a.runs):
        for log in ((False, True) if r % 2 == 0 else (True, False)):
            res.setdefault(f"log {'on' if log else 'off'}", []).append(_run(x, n, log, a.capacity, a.iters))
    drain = [_drain(x, n, a.capacity) for _ in range(a.runs)]
    print(json.dumps({"gpu": gpu, "stereo_instances": n, "nframes": nf, "iters": a.iters, "windows_per_timing": (a.iters + 20) * nf / WINDOW,
                      "capacity": a.capacity, "us_per_block": res, "ms_per_full_drain": drain}))


if __name__ == "__main__":
    main()
