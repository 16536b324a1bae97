"""Cost of the spectrum bank's LTAS plane (b200m_spec_ltas_enable): 4096 stereo instances, 1024-frame blocks (C4), 48 kHz, device
path (b200m_spec_process_device, called directly with its arguments prepared beforehand), in exact mode and in B200M_PREC_FMA, plane
off against plane on.  Each figure is the CUDA-event time per block over --iters blocks after 20 warm-up blocks; every case is taken
--runs times, off and on alternating and swapping order each run.  The GPU's name and power limit are read in the same call and
printed with the results (one JSON line).

    python meters.lv2_b200/host/spec_ltas_cost.py [--n-inst 4096] [--nframes 1024] [--iters 300] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import meters_lv2_b200 as B  # noqa: E402


def _time(fn, iters):
    for _ in range(20):
        B._ck(fn())
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) / iters * 1e3, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-inst", type=int, default=4096)
    ap.add_argument("--nframes", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    n, nf = a.n_inst, a.nframes
    x = (torch.rand(2 * n, nf, device="cuda") * 2 - 1) * 0.5
    p, s, _, _ = B._dev_ptr(x)
    st = B._stream_ptr(None)
    L = B.lib()
    out = {"gpu": gpu, "n_inst": n, "nframes": nf, "us_per_block": {}}
    for mode, prec in (("exact", B.PREC_EXACT), ("tolerance", B.PREC_FMA)):
        res = {"off": [], "on": []}
        for r in range(a.runs):
            for plane in (("off", "on") if r % 2 == 0 else ("on", "off")):
                g = B.Spectr30(n, 2)
                g.set_precision(prec)
                if plane == "on":
                    g.ltas_enable()
                res[plane].append(_time(lambda: L.b200m_spec_process_device(g.h, p, s, nf, 1.0, -4.0, st), a.iters))
                g.close()
        out["us_per_block"][mode] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
