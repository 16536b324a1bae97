"""The EBUr128 cycle's fused K-weighting + true-peak kernel (r128_fused_kernel, csrc/tpk.cu).

In tolerance mode, on the device path, for aligned blocks with nfram % 4 == 0 whose chunk list fits one K1 launch, a bank of at
least R128F_MIN_CH channels runs ONE kernel in place of K1 + tpmax_tc_kernel.  Every case drives the fused bank beside:
 * a PREC_EXACT bank on the same input (K1 + tpmax_kernel): the nine EBU floats and both histograms must be bit-identical;
 * the sliced host path in tolerance mode (each slice runs tpmax_tc_kernel): tp_max must be bit-identical;
and, on a subset of instances, the reference's own TruePeakdsp: tp_max within 1e-4 dB.
"""
import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
FS = 48000.0
R128F_MIN_CH = 10240                         # csrc/tpk.cu
HAVE_REF = O.available("reference")


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _signal(rng, n_inst, n, t0, fs=FS):
    """stereo program: per-instance level (-70..0 dBFS) that moves every few blocks, noise + a tone, some silent instances"""
    lvl = 10.0 ** (rng.uniform(-3.5, 0.0, size=(n_inst, 1)) * (1.0 + 0.3 * np.sin(t0 / fs + np.arange(n_inst)[:, None])))
    lvl[::97] = 0.0
    tt = (t0 + np.arange(n)) / fs
    x = rng.standard_normal((2 * n_inst, n)).astype(np.float32) * 0.25
    x += 0.5 * np.sin(2 * np.pi * (200.0 + 7.0 * np.arange(2 * n_inst)[:, None]) * tt).astype(np.float32)
    return (x * np.repeat(lvl, 2, axis=0)).astype(np.float32)


class _Trio:
    """fused-candidate bank (device, tolerance), exact bank (device), host-path bank (tolerance), optionally an oracle subset"""

    def __init__(self, n_inst, fs=FS, n_ref=0):
        import meters_lv2_b200 as B
        self.B, self.n_inst = B, n_inst
        self.fused, self.exact, self.host = (B.EBUr128(n_inst, fs, True) for _ in range(3))
        for b in (self.fused, self.host):
            b.set_precision(B.PREC_FMA)
        self.banks = (self.fused, self.exact, self.host)
        self.control(B.EBUr128.START)
        self.n_ref = n_ref if HAVE_REF else 0
        if self.n_ref:
            self.ot = O.TruePeak(2 * self.n_ref, fs)
            self.tpmax = np.full(self.n_ref, -np.inf, np.float32)

    def control(self, cmd, inst=-1):
        for b in self.banks:
            b.control(cmd, inst)

    def set_dbtp(self, on):
        for b in self.banks:
            b.set_dbtp(on)
        self.dbtp = on

    def run(self, x_dev, x_host):
        import torch
        B = self.B
        l0 = B.launch_count(); self.fused.run(x_dev); torch.cuda.synchronize(); lf = B.launch_count() - l0
        l0 = B.launch_count(); self.exact.run(x_dev); torch.cuda.synchronize(); le = B.launch_count() - l0
        self.host.run(x_host)
        if self.n_ref:
            if getattr(self, "dbtp", True):
                self.ot.process(np.ascontiguousarray(x_host[:2 * self.n_ref]), mode=1)
                m, _ = self.ot.read()
                v = np.maximum(m[0::2], m[1::2])
                with np.errstate(divide="ignore"):
                    self.tpmax = np.maximum(self.tpmax, np.where(v == 0, -np.inf, 20.0 * np.log10(v.astype(np.float64))).astype(np.float32))
            else:
                self.tpmax[:] = -np.inf
        return lf, le

    def check(self, tag, hist_every=37):
        rf, tf = self.fused.results()
        re, _ = self.exact.results()
        _, th = self.host.results()
        assert rf.tobytes() == re.tobytes(), tag
        bad = np.nonzero(u32(tf) != u32(th))[0]
        assert bad.size == 0, (tag, bad[:5], tf[bad[:3]], th[bad[:3]])
        for i in range(0, self.n_inst, hist_every):
            hf, sf = self.fused.histogram(i); he, se = self.exact.histogram(i)
            assert np.array_equal(hf, he) and np.array_equal(sf, se), (tag, i)
        if self.n_ref:
            fin = np.isfinite(self.tpmax)
            assert np.array_equal(np.isfinite(tf[:self.n_ref]), fin), tag
            if fin.any():
                assert np.abs(tf[:self.n_ref][fin].astype(np.float64) - self.tpmax[fin]).max() <= 1e-4, tag
        return rf, tf


def _ring(n_inst, n, nblk, seed, fs=FS):
    rng = np.random.default_rng(seed)
    return [_signal(rng, n_inst, n, i * n, fs) for i in range(nblk)]


def test_headline_shape_strided_ring():
    """8192 stereo instances, 1024-frame blocks read from a strided device ring (the bench's layout), 480 blocks so that the
    integrated loudness, S maxima and the loudness range are live; one fused kernel replaces K1 + the FIR in every cycle"""
    import torch
    n_inst, nf, R = 8192, 1024, 4
    host = _ring(n_inst, nf, R, seed=1)
    ring = torch.from_numpy(np.concatenate(host, axis=1)).cuda()
    tri = _Trio(n_inst, n_ref=24)
    for b in range(480):
        s = b % R
        lf, le = tri.run(ring[:, s * nf:(s + 1) * nf], host[s])
        assert le - lf == 1, (b, lf, le)                       # K1 + tpmax_kernel -> one kernel
        if b in (0, 1, 2, 100, 479):
            tri.check(b)
    r, _ = tri.fused.results()
    assert (r["integrated"] > -200).mean() > 0.9 and (r["range_max"] > -200).mean() > 0.9


@pytest.mark.parametrize("n_inst", [R128F_MIN_CH // 2 - 1, R128F_MIN_CH // 2, R128F_MIN_CH // 2 + 1, 2 * 8192 + 5])
def test_crossover_and_ragged_slabs(n_inst):
    """just below / at / above the crossover bank size, and slab counts that are not a multiple of 128 channels"""
    import torch
    host = _ring(n_inst, 1024, 3, seed=n_inst)
    tri = _Trio(n_inst, n_ref=8)
    for b in range(12):
        lf, le = tri.run(torch.from_numpy(host[b % 3]).cuda(), host[b % 3])
        assert le - lf == (1 if 2 * n_inst >= R128F_MIN_CH else 0), (b, lf, le)
    tri.check(n_inst)


def test_block_lengths_and_fragment_edges():
    """blocks of 1024, 1000, 64, 4 and 8192 frames: partial last stages, a block inside stage 0 (history in the same row), fragment
    edges (every 2400 frames) inside a stage, and ragged lengths (nfram % 4 != 0) that fall back to the two-kernel cycle"""
    import torch
    n_inst = 6400
    tri = _Trio(n_inst, n_ref=8)
    rng = np.random.default_rng(5)
    sched = [1024, 1000, 64, 4, 8192, 1024, 4, 4, 1000, 8192, 1022, 64, 1024] * 2
    t0 = 0
    for i, n in enumerate(sched):
        x = _signal(rng, n_inst, n, t0); t0 += n
        lf, le = tri.run(torch.from_numpy(x).cuda(), x)
        assert le - lf == (1 if n % 4 == 0 else 0), (i, n, lf, le)
        tri.check((i, n))


def test_low_rate_chunk_overflow_falls_back():
    """a 4 kHz bank: 1024-frame blocks fit one K1 launch (fused), 8192-frame blocks cut into more than 32 chunks (fallback)"""
    import torch
    n_inst, fs = 6400, 4000.0
    tri = _Trio(n_inst, fs=fs, n_ref=8)
    rng = np.random.default_rng(6)
    t0 = 0
    for i, n in enumerate([1024, 8192, 1024, 8192, 8192, 1024]):
        x = _signal(rng, n_inst, n, t0, fs); t0 += n
        lf, le = tri.run(torch.from_numpy(x).cuda(), x)
        assert le - lf == (1 if n == 1024 else 0), (i, n, lf, le)
        tri.check((i, n))


def test_controls_dbtp_snapshot_restore():
    """START / PAUSE / RESET per instance and bank-wide, a slot CLEAR, dBTP toggled, and snapshot / restore across fused cycles"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    n_inst = 6400
    host = _ring(n_inst, 1024, 4, seed=7)
    dev = [torch.from_numpy(h).cuda() for h in host]
    tri = _Trio(n_inst)                                    # per-instance RESET / CLEAR: no oracle subset here
    script = {3: [(E.PAUSE, 5), (E.PAUSE, 6400 - 1)], 6: [(E.RESET, 7)], 9: [(E.START, 5)], 12: [("clear", 130)], 15: [("dbtp", 0)],
              18: [("dbtp", 1)], 21: [(E.RESET, -1)], 24: [(E.START, -1)]}
    snap = None
    for b in range(40):
        for cmd, inst in script.get(b, []):
            if cmd == "clear":
                tri.control(5, inst)                           # B200M_R128_CLEAR: a fresh instance in this slot
            elif cmd == "dbtp":
                tri.set_dbtp(bool(inst))
            else:
                tri.control(cmd, inst)
        tri.run(dev[b % 4], host[b % 4])
        if b % 3 == 2:
            tri.check(b)
        if b == 27:
            snap = tri.fused.snapshot()
    first, tp1 = tri.fused.results()
    tri.fused.restore(snap)
    for b in range(28, 40):
        tri.fused.run(dev[b % 4])
    again, tp2 = tri.fused.results()
    assert first.tobytes() == again.tobytes() and u32(tp1).tobytes() == u32(tp2).tobytes()


def test_nonfinite_rows():
    """NaN and Inf rows and single samples: the maxima ignore NaN outputs like the reference, |Inf| is seen through phase 0"""
    import torch
    n_inst = 6400
    rng = np.random.default_rng(9)
    tri = _Trio(n_inst, n_ref=0)
    for b in range(8):
        x = _signal(rng, n_inst, 1024, b * 1024)
        x[3] = np.nan
        x[10, 17] = np.inf
        x[200 + b, 1023 - b] = -np.inf
        x[500, 64 * b + 5] = np.nan
        x[12799 - 2 * b] = np.nan
        tri.run(torch.from_numpy(x).cuda(), x)
        tri.check(b)
