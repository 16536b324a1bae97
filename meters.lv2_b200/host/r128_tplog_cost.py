"""Cost of the loudness log's dBTP plane (b200m_r128_log_enable) in the EBUr128 cycle, stereo, dBTP on, tolerance and exact mode,
device path:
  (a) b200m_r128_run_device per 1024-frame block with the log off, the loudness-only log (b200m_ebu_log_enable) and the log with the
      dBTP plane, capacity 1200 points = 60 s, the three alternating;
  (b) one b200m_r128_log_drain of every instance's full log (8192 x 1200 points of six fields): the drain kernel and the
      device-to-host copy into pageable memory, as EBUr128.log_drain does it.
(a) is a CUDA-event time per block over --iters blocks, (b) a host clock around the synchronous drain; every figure is taken --runs
times.  The GPU's name and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/r128_tplog_cost.py [--instances 8192] [--nframes 1024] [--iters 300] [--runs 3] [--capacity 1200]
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

PREC = {"tolerance": B.PREC_FMA, "exact": B.PREC_EXACT}
LOGS = ("off", "loudness", "loudness+dbtp")


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


def _cycle(x, n, mode, log, cap, iters):
    bk = B.EBUr128(n, 48000.0, True)
    bk.set_precision(PREC[mode])
    bk.control(B.EBUr128.START)
    if log != "off":
        bk.log_enable(cap, dbtp=log == "loudness+dbtp")
    t = _events(lambda: bk.run(x), iters)
    bk.close()
    return t


def _drain(x, n, cap):
    """ms of one drain of a full log with the dBTP plane: cap points of every instance (written by cap fragments of input)"""
    bk = B.EBUr128(n, 48000.0, True)
    bk.control(B.EBUr128.START)
    bk.log_enable(cap, dbtp=True)
    for _ in range(-(-cap * 2400 // x.shape[1])):
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
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--capacity", type=int, default=1200)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    n, nf = a.instances, a.nframes
    x = (torch.rand(2 * n, nf, device="cuda") * 2 - 1) * 0.5
    res = {}
    for r in range(a.runs):
        for mode in (PREC if r % 2 == 0 else list(PREC)[::-1]):
            for log in (LOGS[r % 3:] + LOGS[:r % 3]):          # each run starts with another case
                res.setdefault(f"{mode} log {log}", []).append(_cycle(x, n, mode, log, a.capacity, a.iters))
    drain = [_drain(x, n, a.capacity) for _ in range(a.runs)]
    print(json.dumps({"gpu": gpu, "stereo_instances": n, "nframes": nf, "capacity": a.capacity, "us_per_block": res,
                      "ms_per_full_drain": drain}))


if __name__ == "__main__":
    main()
