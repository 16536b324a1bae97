"""Cost of albums (b200m_*_group_reduce / b200m_*_group_finish) for a bank of 8192 stereo instances whose histograms hold --seconds
of noise at a level drawn per instance and block (about -60 .. 0 dBFS):
  ebu   album loudness beside the whole-mix reduce and finish (b200m_ebu_mix_*, case "mix"), 20 s, 200 calls per timing; the
        reduce reads n_inst x 1508 x 4 bytes of histograms;
  dr14  album DR, 60 s, 50 calls per timing; the reduce (the zeroing of the rows, the reduce kernel and the peaks kernel) reads
        n_inst x 2 x 8000 x 4 bytes.
Album layouts: G = 1, 64, 1024, 8192 (album of instance i: i * G // n_inst) and a skewed assignment (one album of half the bank,
one album per instance for the other half).  Each case is timed as (a) one reduce call (the zeroing of the G output rows and the
kernels): CUDA events over --iters back-to-back calls, and the achieved rate over the histogram read; (b) one reduce + finish call
(the finish copies the G results to the host and synchronises): a host clock over --iters calls.  Both entry points are called
through ctypes with prepared arguments, as bench.py calls the process entry points.  Each figure is taken --runs times, the cases
alternating; every album layout's rows are checked to sum to the whole (the whole-mix vector; for dr14, the G = 1 row).  The
GPU's name and power limit are read in the same call and printed with the results (one JSON line).

    python meters.lv2_b200/host/group_cost.py [--banks ebu,dr14] [--instances 8192] [--seconds S] [--iters N] [--runs 3]
"""
import ctypes as C
import json

import numpy as np
import torch

import _cost
from _cost import B


def _fill(n, seconds, nfram, feed):
    """feed the bank `seconds` of stereo noise, nfram frames per block, at a level drawn per instance and block; returns the last
    block and its levels, which the caller holds through its timings: where the caching allocator then puts the album rows is
    where it put them for the figures in DESIGN.md (freeing the block moves the G = 1 reduce by about 2 %)"""
    gen = torch.Generator(device="cuda"); gen.manual_seed(0)
    for _ in range(int(seconds * 48000) // nfram):
        lvl = 10.0 ** (torch.rand(n, 1, device="cuda", generator=gen) * -3.0)
        x = (torch.rand(2 * n, nfram, device="cuda", generator=gen) * 2 - 1) * lvl.repeat_interleave(2, 0)
        feed(x)
    torch.cuda.synchronize()
    return x, lvl


def _layouts(n):
    lay = {f"G={g}": (np.arange(n) * g // n, g) for g in (1, 64, 1024, 8192)}
    half = n // 2
    lay["skewed"] = (np.concatenate([np.zeros(half, np.int64), 1 + np.arange(n - half)]), 1 + n - half)
    return lay


def _measure(runs, iters, warmup, cases, n, seconds, read_mb, nonzero):
    """cases: name -> (reduce, reduce + finish) closures; -> the bank's JSON object"""
    red, both = {}, {}
    for r in range(runs):
        for name in _cost.alternate(cases, r):
            reduce, finish = cases[name]
            red.setdefault(name, []).append(_cost.events(reduce, iters, warmup))
            both.setdefault(name, []).append(_cost.host_clock(finish, iters, warmup))
    gbs = {k: [round(read_mb / t * 1e3, 1) for t in v] for k, v in red.items()}              # MB / us = TB/s
    return {"stereo_instances": n, "seconds": seconds, "hist_read_MB": round(read_mb, 1), "nonzero_words_per_instance": nonzero,
            "reduce_us": red, "reduce_GBps": gbs, "reduce_finish_us": both}


def ebu(a):
    n, seconds = a.instances, a.seconds or 20.0
    L, st = B.lib(), B._stream_ptr(None)
    bank = B.Ebu_r128_proc(n, 2)
    bank.integr_start()
    last = _fill(n, seconds, 1024, bank.process)  # noqa: F841
    mix = torch.zeros(B.MIX_WORDS, dtype=torch.int32, device="cuda")
    mp, out5 = C.c_void_p(mix.data_ptr()), np.empty(5, np.float32)
    bank.mix_reduce(mix)
    prepared = {}
    for name, (groups, g) in _layouts(n).items():
        d = torch.empty((g, B.MIX_WORDS), dtype=torch.int32, device="cuda")
        bank.group_reduce(groups, d)
        assert torch.equal(d.sum(0, dtype=torch.int64), mix.long()), name          # every instance is in one album
        prepared[name] = (np.ascontiguousarray(groups.astype(np.uint32)), g, d, np.empty((g, 5), np.float32))
    rows = prepared["G=8192"][2] if n == 8192 else None
    nonzero = None if rows is None else round(float((rows != 0).sum().item()) / n, 1)

    def case(g32, g, d, o):
        gp, dp, op = B._np_ptr(g32), C.c_void_p(d.data_ptr()), B._np_ptr(o)

        def reduce():
            B._ck(L.b200m_ebu_group_reduce(bank.h, gp, g, dp, st))

        def finish():
            reduce()
            B._ck(L.b200m_ebu_group_finish(bank.h, dp, g, op, st))
        return reduce, finish

    def mix_reduce():
        B._ck(L.b200m_ebu_mix_reduce(bank.h, mp, st))

    def mix_finish():
        mix_reduce()
        B._ck(L.b200m_ebu_mix_finish(bank.h, mp, B._np_ptr(out5), st))

    cases = {name: case(*p) for name, p in prepared.items()}
    cases["mix"] = (mix_reduce, mix_finish)
    return _measure(a.runs, a.iters or 200, 10, cases, n, seconds, n * B.MIX_WORDS * 4 / 1e6, nonzero)


def dr14(a):
    n, nch, seconds = a.instances, 2, a.seconds or 60.0
    L, st = B.lib(), B._stream_ptr(None)
    bank = B.DR14(n, nch, 48000.0, True)
    last = _fill(n, seconds, 8192, bank.run)  # noqa: F841
    words = B.dr14_group_words(nch)
    prepared, total = {}, None
    for name, (groups, g) in _layouts(n).items():
        d = torch.empty((g, words), dtype=torch.int32, device="cuda")
        p = torch.empty((g, nch, 3), dtype=torch.float32, device="cuda")
        bank.group_reduce(groups, d, p)
        s = d.sum(0, dtype=torch.int64)
        total = s if total is None else total
        assert torch.equal(s, total), name                                  # every instance is in one album
        prepared[name] = (np.ascontiguousarray(groups.astype(np.uint32)), g, d, p, np.empty(g, B.DR14_ALBUM_DTYPE))
    rows = prepared["G=8192"][2] if n == 8192 else None
    nonzero = None if rows is None else round(float((rows[:, :-2] != 0).sum().item()) / n, 1)

    def case(g32, g, d, p, o):
        gp, dp, pp, op = B._np_ptr(g32), C.c_void_p(d.data_ptr()), C.c_void_p(p.data_ptr()), B._np_ptr(o)

        def reduce():
            B._ck(L.b200m_dr14_group_reduce(bank.h, gp, g, dp, pp, st))

        def finish():
            reduce()
            B._ck(L.b200m_dr14_group_finish(bank.h, dp, pp, 1, g, op, st))
        return reduce, finish

    cases = {name: case(*p) for name, p in prepared.items()}
    return _measure(a.runs, a.iters or 50, 5, cases, n, seconds, n * nch * 8000 * 4 / 1e6, nonzero)


BANKS = {"ebu": ebu, "dr14": dr14}


def main():
    ap = _cost.parser(__doc__, banks=BANKS, instances=8192, iters=None, runs=3)
    ap.add_argument("--seconds", type=float, help="seconds of noise in the histograms (default: each bank's own)")
    a = ap.parse_args()
    out = {"gpu": _cost.gpu()}
    for name in a.banks.split(","):
        out[name] = BANKS[name](a)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
