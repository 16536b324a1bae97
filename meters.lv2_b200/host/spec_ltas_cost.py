"""Cost of the spectrum bank's LTAS plane (b200m_spec_ltas_enable): 4096 stereo instances, 1024-frame blocks (C4), 48 kHz, device
path (b200m_spec_process_device, called directly with its arguments prepared beforehand), in exact mode and in B200M_PREC_FMA, plane
off against plane on.  Each figure is the CUDA-event time per block over --iters blocks after 20 warm-up blocks; every case is taken
--runs times, off and on alternating and swapping order each run.  The GPU's name and power limit are read in the same call and
printed with the results (one JSON line).

    python meters.lv2_b200/host/spec_ltas_cost.py [--instances 4096] [--nframes 1024] [--iters 300] [--runs 3]
"""
import json

import _cost
from _cost import B


def main():
    a = _cost.parser(__doc__, instances=4096, nframes=1024, iters=300, runs=3).parse_args()
    gpu = _cost.gpu()
    n, nf = a.instances, a.nframes
    x = _cost.noise(2 * n, nf)
    p, s, _, _ = B._dev_ptr(x)
    st = B._stream_ptr(None)
    L = B.lib()
    out = {"gpu": gpu, "n_inst": n, "nframes": nf, "us_per_block": {}}
    for mode, prec in (("exact", B.PREC_EXACT), ("tolerance", B.PREC_FMA)):
        res = {"off": [], "on": []}
        for r in range(a.runs):
            for plane in _cost.alternate(("off", "on"), r):
                g = B.Spectr30(n, 2)
                g.set_precision(prec)
                if plane == "on":
                    g.ltas_enable()
                res[plane].append(_cost.events(lambda: L.b200m_spec_process_device(g.h, p, s, nf, 1.0, -4.0, st), a.iters, 20))
                g.close()
        out["us_per_block"][mode] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
