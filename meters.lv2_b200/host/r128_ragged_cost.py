"""Cost of ragged blocks in the EBUr128 cycle (b200m_r128_run_ragged_device), stereo, dBTP on, tolerance and exact mode:
  (a) b200m_r128_run_device against b200m_r128_run_ragged_device with every length equal to nfram (the same call);
  (b) blocks in which 1 % / 50 % of the instances end early (a random length below nfram);
  (c) b200m_r128_run_device in steady state after ragged blocks have scattered the instances over >= 64 fragment phase classes;
  (d) programme_loudness throughput in clip-seconds per second, clips of 20-60 s against the same number of clips all 60 s long
      (one device block reused for every offset, so that the figure is the metering alone).
(a)-(c) are CUDA-event times per block over --iters blocks; every figure is taken --runs times, the modes alternating.  The GPU's
name and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/r128_ragged_cost.py [--instances 8192] [--nframes 1024] [--iters 300] [--runs 3]
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

PREC = {"tolerance": B.PREC_FMA, "exact": B.PREC_EXACT}


def _bank(n, mode):
    bk = B.EBUr128(n, 48000.0, True)
    bk.set_precision(PREC[mode])
    bk.control(B.EBUr128.START)
    return bk


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


def _one(x, n, nf, mode, iters, rng):
    out = {}
    full = np.full(n, nf, np.uint32)
    bk = _bank(n, mode)
    out["a plain"] = _events(lambda: bk.run(x), iters)
    out["a ragged all nfram"] = _events(lambda: bk.run(x, lengths=full), iters)
    for pct in (1, 50):
        lens = full.copy()
        idx = rng.choice(n, size=n * pct // 100, replace=False)
        lens[idx] = rng.integers(0, nf, size=idx.size)
        out[f"b {pct}% end early"] = _events(lambda: bk.run(x, lengths=lens), iters)
    bk.close()
    bk = _bank(n, mode)
    for k in range(64):                        # 64 blocks in which one instance in 64 is one frame short: >= 64 phase classes
        lens = full.copy(); lens[k::64] = nf - 1 - k
        bk.run(x, lengths=lens)
    out["c plain after scatter"] = _events(lambda: bk.run(x), iters)
    bk.close()
    return out


def _programme(x, n, nf, lengths):
    get = lambda off, m: x[:, :m]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    B.programme_loudness(get, lengths, 48000.0, block=nf, precision=B.PREC_FMA)
    torch.cuda.synchronize()
    return round(float(np.sum(lengths)) / 48000.0 / (time.perf_counter() - t0), 1)


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
    res = {}
    for r in range(a.runs):
        for mode in (PREC if r % 2 == 0 else list(PREC)[::-1]):
            for k, v in _one(x, n, nf, mode, a.iters, rng).items():
                res.setdefault(f"{mode} {k}", []).append(v)
    mixed = rng.integers(20 * 48000, 60 * 48000, size=n)
    for r in range(a.runs):
        res.setdefault("d clips 20-60 s", []).append(_programme(x, n, nf, mixed))
        res.setdefault("d clips all 60 s", []).append(_programme(x, n, nf, np.full(n, 60 * 48000)))
    print(json.dumps({"gpu": gpu, "stereo_instances": n, "nframes": nf, "us_per_block": {k: v for k, v in res.items() if not k.startswith("d ")},
                      "clip_seconds_per_second": {k: v for k, v in res.items() if k.startswith("d ")}}))


if __name__ == "__main__":
    main()
