"""Cost of the point logs, stereo, 48 kHz, device path, 8192 instances x 1024-frame blocks:
  r128  the EBUr128 cycle (b200m_r128_run_device), dBTP on, tolerance and exact mode, with the log off, the loudness-only log
        (b200m_ebu_log_enable) and the log with the dBTP plane (b200m_r128_log_enable), capacity 1200 points = 60 s; and one
        drain of every instance's full log (8192 x 1200 points), loudness only (b200m_ebu_log_drain) and with the dBTP plane
        (b200m_r128_log_drain, six fields);
  dr14  b200m_dr14_run_device, DR mode, with the window log (b200m_dr14_log_enable) off and on, capacity 16 points = 48 s,
        timed over 600 blocks: 3 s windows and more of audio, so that the blocks in which windows close (and the log writes its
        points) are in the timing; and one b200m_dr14_log_drain of every instance's full log (8192 x 16 points).
A drain is the drain kernel and the device-to-host copy into pageable memory, as the banks' log_drain does it.  Block times are
CUDA events per block over --iters blocks, drains a host clock around the synchronous drain; every figure is taken --runs times,
the cases alternating.  The GPU's name and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/log_cost.py [--banks r128,dr14] [--instances 8192] [--nframes 1024] [--iters N] [--runs 3]
                                            [--capacity N]
"""
import json

import _cost
from _cost import B

RATE = 48000.0
PREC = {"tolerance": B.PREC_FMA, "exact": B.PREC_EXACT}
LOGS = ("off", "loudness", "loudness+dbtp")
FRAGMENT = 2400                 # frames of one 50 ms fragment: one loudness point
WINDOW = 144001                 # rintf (3 * 48000) + 1 frames: one DR point


def _drain(bk, x, cap, frames):
    """ms of one drain of a full log: cap points of every instance, written by cap periods of `frames` frames of input"""
    for _ in range(-(-cap * frames // x.shape[1])):
        bk.run(x)
    got = []
    t = _cost.host_clock(lambda: got.append(bk.log_drain()))
    assert (got[0][1] == cap).all()
    bk.close()
    return round(t / 1e3, 2)


def r128(a, x):
    n, iters, cap = a.instances, a.iters or 300, a.capacity or 1200

    def bank(log, mode=None):
        bk = B.EBUr128(n, RATE, True)
        if mode is not None:
            bk.set_precision(PREC[mode])
        bk.control(B.EBUr128.START)
        if log != "off":
            bk.log_enable(cap, dbtp=log == "loudness+dbtp")
        return bk

    def cycle(mode, log):
        bk = bank(log, mode)
        t = _cost.events(lambda: bk.run(x), iters, 20)
        bk.close()
        return t

    res, drain = {}, {}
    for r in range(a.runs):
        for mode in _cost.alternate(PREC, r):
            for log in _cost.alternate(LOGS, r):
                res.setdefault(f"{mode} log {log}", []).append(cycle(mode, log))
    for r in range(a.runs):
        for log in _cost.alternate(LOGS[1:], r):
            drain.setdefault(log, []).append(_drain(bank(log), x, cap, FRAGMENT))
    return {"stereo_instances": n, "nframes": a.nframes, "capacity": cap, "us_per_block": res, "ms_per_full_drain": drain}


def dr14(a, x):
    n, iters, cap = a.instances, a.iters or 600, a.capacity or 16

    def bank(log):
        bk = B.DR14(n, 2, RATE, True)
        if log == "on":
            bk.log_enable(cap)
        return bk

    def run(log):
        bk = bank(log)
        t = _cost.events(lambda: bk.run(x), iters, 20)
        bk.close()
        return t

    res = {}
    for r in range(a.runs):
        for log in _cost.alternate(("off", "on"), r):
            res.setdefault(f"log {log}", []).append(run(log))
    drain = [_drain(bank("on"), x, cap, WINDOW) for _ in range(a.runs)]
    return {"stereo_instances": n, "nframes": a.nframes, "iters": iters, "windows_per_timing": (iters + 20) * a.nframes / WINDOW,
            "capacity": cap, "us_per_block": res, "ms_per_full_drain": drain}


BANKS = {"r128": r128, "dr14": dr14}


def main():
    ap = _cost.parser(__doc__, banks=BANKS, instances=8192, nframes=1024, iters=None, runs=3)
    ap.add_argument("--capacity", type=int, help="log points per instance (default: each bank's own)")
    a = ap.parse_args()
    out = {"gpu": _cost.gpu()}
    for name in a.banks.split(","):
        out[name] = BANKS[name](a, _cost.noise(2 * a.instances, a.nframes))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
