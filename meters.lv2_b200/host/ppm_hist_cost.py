"""Cost of the needle-meter bank's histogram plane (b200m_ppm_hist_enable): IEC II with 16384 meters, M/S with 8192 pairs and VU with
16384 meters, 1024-frame blocks, 48 kHz, device path (b200m_ppm_process_device, called directly with its arguments prepared
beforehand), plane off against plane on (limit 0 dB).  The input is uniform noise in [-0.5, 0.5), so every needle wanders over a few
bins and some readings pass the limit.  Each figure is the CUDA-event time per block over --iters blocks after 20 warm-up blocks;
every case is taken --runs times, off and on alternating and swapping order each run.  The GPU's name and power limit are read in
the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/ppm_hist_cost.py [--nframes 1024] [--iters 300] [--runs 3]
"""
import json

import _cost
from _cost import B

CASES = (("iec2", B.PPM_IEC2, 16384), ("ms", B.PPM_MS, 8192), ("vu", B.PPM_VU, 16384))


def main():
    ap = _cost.parser(__doc__, nframes=1024, iters=300, runs=3)
    a = ap.parse_args()
    gpu = _cost.gpu()
    nf = a.nframes
    st = B._stream_ptr(None)
    L = B.lib()
    out = {"gpu": gpu, "nframes": nf, "us_per_block": {}}
    for name, kind, n in CASES:
        x = _cost.noise(2 * n if kind == B.PPM_MS else n, nf)
        p, s, _, _ = B._dev_ptr(x)
        res = {"units": n, "off": [], "on": []}
        for r in range(a.runs):
            for plane in _cost.alternate(("off", "on"), r):
                g = B.NeedleMeters(n, kind)
                if plane == "on":
                    g.hist_enable()
                res[plane].append(_cost.events(lambda: L.b200m_ppm_process_device(g.h, p, s, nf, st), a.iters, 20))
                g.close()
        out["us_per_block"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
