"""Cost of the phasewheel bank's cross-spectrum plane (b200m_pw_xspec_enable), plane off against plane on, device path
(b200m_pw_process_device, called directly with its arguments prepared beforehand), 48 kHz:
  c5       2048 instances, fft_bins 1024, 1024-frame blocks (C5's shape): an analysis every ~1.9 blocks;
  c5_cor   the same with a correlation bank of 2048 pairs attached (fused feed);
  fb2048   2048 instances, fft_bins 2048 (programme_stereo's default), 1024-frame blocks;
  multi    2048 instances, fft_bins 256, 8192-frame blocks: about four analyses per call, all but the last plane-only.
Each figure is the CUDA-event time per block over --iters blocks after 20 warm-up blocks; every case is taken --runs times, off and
on alternating and swapping order each run.  The GPU's name and power limit are read in the same call and printed with the results
(one JSON line).

    python meters.lv2_b200/host/pw_xspec_cost.py [--instances 2048] [--iters 200] [--runs 3]
"""
import json

import _cost
from _cost import B

CASES = (("c5", 1024, 1024, False), ("c5_cor", 1024, 1024, True), ("fb2048", 2048, 1024, False), ("multi", 256, 8192, False))


def main():
    a = _cost.parser(__doc__, instances=2048, iters=200, runs=3).parse_args()
    gpu = _cost.gpu()
    n = a.instances
    L = B.lib()
    st = B._stream_ptr(None)
    out = {"gpu": gpu, "n_inst": n, "us_per_block": {}}
    for name, bins, nf, cor in CASES:
        x = _cost.noise(2 * n, nf)
        p, s, _, _ = B._dev_ptr(x)
        res = {"off": [], "on": []}
        for r in range(a.runs):
            for plane in _cost.alternate(("off", "on"), r):
                g = B.Phasewheel(n, bins)
                c = None
                if cor:
                    c = B.Stcorrdsp(n)
                    g.attach_cor(c)
                if plane == "on":
                    g.xspec_enable()
                res[plane].append(_cost.events(lambda: L.b200m_pw_process_device(g.h, p, s, nf, 1e-6, None, st), a.iters, 20))
                g.close()
                if c is not None:
                    c.close()
        out["us_per_block"][name] = dict(fft_bins=bins, nframes=nf, **res)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
