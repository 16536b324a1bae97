"""Cost of the correlation bank's histogram plane (b200m_cor_hist_enable): 2048 pairs (the C5 size) and 8192 pairs, 1024-frame
blocks, 48 kHz, tcf 0.3 s, device path (b200m_cor_process_device, called directly with its arguments prepared beforehand), in exact
mode and in B200M_PREC_FMA, plane off against plane on (default -70 dB gate).  The input is independent uniform noise on L and R,
so the readings wander near 0 across a few bins.  With the plane on, tolerance mode runs the exact kernel.  Each figure is the
CUDA-event time per block over --iters blocks after 20 warm-up blocks; every case is taken --runs times, off and on alternating
and swapping order each run.  The GPU's name and power limit are read in the same call and printed with the results (one JSON
line).

    python meters.lv2_b200/host/cor_hist_cost.py [--pairs 2048,8192] [--nframes 1024] [--iters 300] [--runs 3]
"""
import json

import _cost
from _cost import B


def main():
    ap = _cost.parser(__doc__, nframes=1024, iters=300, runs=3)
    ap.add_argument("--pairs", default="2048,8192", help="comma-separated bank sizes (default: %(default)s)")
    a = ap.parse_args()
    gpu = _cost.gpu()
    nf = a.nframes
    st = B._stream_ptr(None)
    L = B.lib()
    out = {"gpu": gpu, "nframes": nf, "us_per_block": {}}
    for n in (int(v) for v in a.pairs.split(",")):
        x = _cost.noise(2 * n, nf)
        p, s, _, _ = B._dev_ptr(x)
        per = {}
        for mode, prec in (("exact", B.PREC_EXACT), ("tolerance", B.PREC_FMA)):
            res = {"off": [], "on": []}
            for r in range(a.runs):
                for plane in _cost.alternate(("off", "on"), r):
                    g = B.Stcorrdsp(n)
                    g.set_precision(prec)
                    if plane == "on":
                        g.hist_enable()
                    res[plane].append(_cost.events(lambda: L.b200m_cor_process_device(g.h, p, s, nf, st), a.iters, 20))
                    g.close()
            per[mode] = res
        out["us_per_block"][str(n)] = per
    print(json.dumps(out))


if __name__ == "__main__":
    main()
