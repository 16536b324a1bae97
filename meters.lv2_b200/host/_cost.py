"""What the cost scripts in this directory share: the GPU's name and power limit, the timers, the order of the cases in each run,
the ragged length draws, the seeded input and the arguments.  The warm-up count is each caller's: every measurement keeps the one
its figures were taken with.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import meters_lv2_b200 as B  # noqa: E402

_HELP = {"runs": "times every case is measured, the case order reversed on every other run",
         "iters": "calls per timing", "nframes": "frames per block", "instances": "instances per bank"}


def parser(doc, banks=None, lib=False, **defaults):
    """an argument parser whose --help prints doc, with --runs, --iters, --nframes and --instances for those of them given a
    default here (None: each bank's own), --banks (a comma-separated subset of `banks`) and --lib (repeatable: the builds of
    libb200meters.so to alternate; default this tree's)"""
    ap = argparse.ArgumentParser(description=doc, formatter_class=argparse.RawDescriptionHelpFormatter)
    for k, d in defaults.items():
        ap.add_argument("--" + k, type=int, default=d, help=_HELP[k] + (" (default: each bank's own)" if d is None else " (default: %(default)s)"))
    if banks:
        ap.add_argument("--banks", default=",".join(banks), help="comma-separated, from %(default)s")
    if lib:
        ap.add_argument("--lib", action="append", help="a build of libb200meters.so, repeatable (default: this tree's)")
    return ap


def gpu():
    """the GPU's name and power limit, printed beside every figure"""
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def noise(rows, nframes):
    """the input block: uniform noise in [-0.5, 0.5) on the device, drawn after torch.manual_seed(0)"""
    torch.manual_seed(0)
    return (torch.rand(rows, nframes, device="cuda") * 2 - 1) * 0.5


def alternate(cases, r):
    """the cases of run r: in their order on even runs, reversed on odd ones"""
    cases = list(cases)
    return cases if r % 2 == 0 else cases[::-1]


def events(fn, iters, warmup, host=False):
    """µs per call of fn by CUDA events over iters back-to-back calls, after warmup calls (a non-zero return is a C entry
    point's error code) and a synchronise; host=True also returns the host's wall µs per call in the same loop"""
    for _ in range(warmup):
        B._ck(fn() or 0)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    wall = time.perf_counter() - t0
    b.record()
    torch.cuda.synchronize()
    dev = round(a.elapsed_time(b) / iters * 1e3, 2)
    return (dev, round(wall / iters * 1e6, 2)) if host else dev


def host_clock(fn, iters=1, warmup=0):
    """µs per call of fn by the host clock over iters calls, after warmup calls and a synchronise; fn ends in a synchronise of
    its own (a finish, a drain)"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return round((time.perf_counter() - t0) / iters * 1e6, 2)


def ragged_forms(n, nfram, rng, ab=False):
    """the four forms of a ragged timing of n rows: the plain call (None), every length nfram, and 1 % / 50 % of the rows ending
    early at a random length below nfram, drawn from rng in that order.  ab=True labels them as the scripts that time more parts
    do: (a) the plain and the equal-length call, (b) rows ending early"""
    a, b = ("a ", "b ") if ab else ("", "")
    full = np.full(n, nfram, np.uint32)
    forms = {a + "plain": None, a + "ragged all nfram": full}
    for pct in (1, 50):
        lens = full.copy()
        idx = rng.choice(n, size=max(1, n * pct // 100), replace=False)
        lens[idx] = rng.integers(0, nfram, size=idx.size)
        forms[f"{b}{pct}% end early"] = lens
    return forms
