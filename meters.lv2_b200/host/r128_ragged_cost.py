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
import json
import time

import numpy as np
import torch

import _cost
from _cost import B

PREC = {"tolerance": B.PREC_FMA, "exact": B.PREC_EXACT}


def _bank(n, mode):
    bk = B.EBUr128(n, 48000.0, True)
    bk.set_precision(PREC[mode])
    bk.control(B.EBUr128.START)
    return bk


def _one(x, n, nf, mode, iters, rng):
    out = {}
    bk = _bank(n, mode)
    for k, lens in _cost.ragged_forms(n, nf, rng, ab=True).items():
        out[k] = _cost.events(lambda: bk.run(x, lengths=lens), iters, 20)
    bk.close()
    bk = _bank(n, mode)
    full = np.full(n, nf, np.uint32)
    for k in range(64):                        # 64 blocks in which one instance in 64 is one frame short: >= 64 phase classes
        lens = full.copy(); lens[k::64] = nf - 1 - k
        bk.run(x, lengths=lens)
    out["c plain after scatter"] = _cost.events(lambda: bk.run(x), iters, 20)
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
    a = _cost.parser(__doc__, instances=8192, nframes=1024, iters=300, runs=3).parse_args()
    gpu = _cost.gpu()
    n, nf = a.instances, a.nframes
    x = _cost.noise(2 * n, nf)
    rng = np.random.default_rng(0)
    res = {}
    for r in range(a.runs):
        for mode in _cost.alternate(PREC, r):
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
