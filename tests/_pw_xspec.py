"""Oracle of the phasewheel bank's cross-spectrum plane (b200m_pw_xspec_enable): float64 restatement from numpy's FFT.

The plane sums, per instance and bin k < fft_bins, |L_k|^2, |R_k|^2 and R_k conj L_k over every analysis the reference's fftx_run
computes (gui/fft.c:308-338, the step loop at :346-360), not only the last one of a call.  This restates that clock per instance:
sps = ceil (rate / 25), each call walked in steps of min (N, remaining) frames, an analysis whenever the step count reaches sps.  An
analysis takes the clip's last N = 2 fft_bins frames, zero-padded on the left (the ring starts zeroed), and forms the terms from
_fftref.spectra.  The bank's fp32 transform is pinned to numpy within |dX| <= EPS max|X| per analysis (test_pw_gpu.py); `bound`
propagates that into each term and sums it over the analyses, so a bank row must lie within bound of the oracle's sums.
"""
import math

import numpy as np

import _fftref as F

EPS = 2e-6


def clock(calls, fft_bins, rate, smps=0):
    """calls: frame counts of one instance's successive calls (0: not called).  Returns (ends, fired): the clip position (frames fed
    so far) at each analysis, and per call 1 if it analysed"""
    N, sps = 2 * int(fft_bins), math.ceil(float(rate) / 25.0)
    pos, ends, fired = 0, [], []
    for n in calls:
        d, f = 0, 0
        while d < n:
            m = min(N, n - d)
            smps += m; pos += m; d += m
            if smps >= sps:
                smps = 0; ends.append(pos); f = 1
        fired.append(f)
    return ends, fired


def analyse(x, ends, fft_bins):
    """the plane row of one stereo clip x [2, T] (float32) whose analyses end at `ends`: dict of sums and bound (float64 [4, fft_bins],
    PW_XSPEC_TERMS order), analyses and skipped (an analysis with a non-finite spectrum adds nothing)"""
    bins, N = int(fft_bins), 2 * int(fft_bins)
    x = np.asarray(x, np.float32)
    sums, bound = np.zeros((4, bins)), np.zeros((4, bins))
    analyses = skipped = 0
    for e in ends:
        fr = np.zeros((2, N), np.float32)
        seg = x[:, max(0, e - N):e]
        fr[:, N - seg.shape[1]:] = seg
        X, _, _ = F.spectra(fr)
        if not np.isfinite(X).all():
            skipped += 1
            continue
        analyses += 1
        L, R = X[0, :bins], X[1, :bins]
        dl, dr = EPS * np.abs(X[0]).max(), EPS * np.abs(X[1]).max()
        lr, li, rr, ri = L.real, L.imag, R.real, R.imag      # the terms as the bank forms them from the parts
        t = np.stack([lr * lr + li * li, rr * rr + ri * ri, rr * lr + ri * li, ri * lr - rr * li])
        sums += t
        al, ar = np.abs(L), np.abs(R)
        bc = ar * dl + al * dr + dl * dr
        bound += np.stack([2 * al * dl + dl * dl, 2 * ar * dr + dr * dr, bc, bc]) + 1e-13 * np.abs(t)
    return dict(sums=sums, bound=bound, analyses=analyses, skipped=skipped)


def bank(x, calls, fft_bins, rate):
    """rows of n instances, x [2n, T], fed calls [C][n] frame counts (instance i's frames of call c follow its earlier ones in its
    rows): (sums [n, 4, bins], bound [n, 4, bins], analyses [n], skipped [n])"""
    calls = np.asarray(calls, np.int64).reshape(len(calls), -1)
    n = calls.shape[1]
    rows = []
    for i in range(n):
        ends, _ = clock(calls[:, i], fft_bins, rate)
        rows.append(analyse(x[2 * i:2 * i + 2], ends, fft_bins))
    return (np.stack([r["sums"] for r in rows]), np.stack([r["bound"] for r in rows]),
            np.array([r["analyses"] for r in rows], np.int64), np.array([r["skipped"] for r in rows], np.int64))
