"""Cost of ragged blocks in the DR-14 bank (b200m_dr14_run_ragged_device), stereo, DR mode, 48 kHz:
  (a) b200m_dr14_run_device against b200m_dr14_run_ragged_device with every length equal to nfram (the same call);
  (b) blocks in which 1 % / 50 % of the instances end early (a random length below nfram).
Each figure is the CUDA-event time per block over --iters blocks, next to the host's wall time per call in the same loop (the
enqueue, the lengths' upload and the phase mirror; the host runs ahead of the device until the launch queue is full, so where
the two agree the host may be the bound).  Every figure is taken --runs times, the forms alternating.  The GPU's name
and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/dr14_ragged_cost.py [--instances 8192] [--nframes 1024] [--iters 300] [--runs 3]
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
        fn()
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
    forms = {"a plain": None, "a ragged all nfram": full}
    for pct in (1, 50):
        lens = full.copy()
        idx = rng.choice(n, size=n * pct // 100, replace=False)
        lens[idx] = rng.integers(0, nf, size=idx.size)
        forms[f"b {pct}% end early"] = lens
    return forms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--instances", type=int, default=8192)
    ap.add_argument("--nframes", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=300)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    n, nf = a.instances, a.nframes
    x = (torch.rand(2 * n, nf, device="cuda") * 2 - 1) * 0.5
    rng = np.random.default_rng(0)
    forms = _forms(n, nf, rng)
    res, host = {}, {}
    for r in range(a.runs):
        for k in (list(forms) if r % 2 == 0 else list(forms)[::-1]):
            bk = B.DR14(n, 2, 48000.0, True)
            lens = forms[k]
            dev, hst = _time((lambda: bk.run(x)) if lens is None else (lambda: bk.run(x, lengths=lens)), a.iters)
            res.setdefault(k, []).append(dev)
            host.setdefault(k, []).append(hst)
            bk.close()
    print(json.dumps({"gpu": gpu, "stereo_instances": n, "nframes": nf, "us_per_block": res, "host_us_per_call": host}))


if __name__ == "__main__":
    main()
