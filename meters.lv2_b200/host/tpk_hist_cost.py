"""Cost of the true-peak / K-meter bank's histogram plane (b200m_tpk_hist_enable): 16384 channels in three banks (true peak + K-meter,
true peak only, K-meter only), exact and tolerance (FMA) precision, 1024-frame blocks, 48 kHz, device path
(b200m_tpk_process_device in process() mode, called directly with its arguments prepared beforehand), plane off against plane on
(limits -1 dBTP and -10 dBFS).  The input is uniform noise in [-0.5, 0.5), so the true-peak readings spread over many bins and some
pass the limit.  With the plane on every block runs the exact 16-channel kernel, in either precision.  Each figure is the CUDA-event
time per block over --iters blocks after 20 warm-up blocks; every case is taken --runs times, off and on alternating and swapping
order each run.  The GPU's name and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/tpk_hist_cost.py [--instances 16384] [--nframes 1024] [--iters 300] [--runs 3]
"""
import json

import _cost
from _cost import B

BANKS = (("tp_km", B.TPK_TRUEPEAK | B.TPK_KMETER), ("tp", B.TPK_TRUEPEAK), ("km", B.TPK_KMETER))
PRECISIONS = (("exact", B.PREC_EXACT), ("fma", B.PREC_FMA))


def main():
    ap = _cost.parser(__doc__, nframes=1024, iters=300, runs=3, instances=16384)
    a = ap.parse_args()
    gpu = _cost.gpu()
    n, nf = a.instances, a.nframes
    st = B._stream_ptr(None)
    L = B.lib()
    x = _cost.noise(n, nf)
    p, s, _, _ = B._dev_ptr(x)
    out = {"gpu": gpu, "channels": n, "nframes": nf, "us_per_block": {}}
    for name, flags in BANKS:
        for pname, prec in PRECISIONS:
            res = {"off": [], "on": []}
            for r in range(a.runs):
                for plane in _cost.alternate(("off", "on"), r):
                    g = B.TruePeakKmeter(n, 48000.0, flags)
                    g.set_precision(prec)
                    if plane == "on":
                        g.hist_enable()
                    res[plane].append(_cost.events(lambda: L.b200m_tpk_process_device(g.h, p, s, nf, B.TP_MODE_PROCESS, st), a.iters, 20))
                    g.close()
            out["us_per_block"]["%s/%s" % (name, pname)] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
