"""GPU: the tolerance modes (B200M_PREC_FMA) at the mastering rates 44.1-192 kHz, and the EBUr128 cycle where a 50 ms fragment is
longer than the largest block.

What the tolerance modes rewrite are recurrences whose memory grows with the rate: the correlation's product filters
(1 / w2 = tcf * fs samples), the K-meter's RMS filter (fs / 9.72) and the spectrum's lowest bands (biquad poles move towards
z = 1).  The reference runs those filters serially in fp32 and its own rounding noise grows with their memory, so every case is
checked twice where it can be: against the reference oracle (its documented tolerance) and against a float64 restatement of the
same linear filters written here with scipy.signal (a bound that does not move with the reference's noise, and would catch a
kernel that is wrong by less than the reference's own error).  Past a product-filter memory of COR_SCAN_MAX_MEMORY samples the
reference's noise alone would break the correlation's 1e-5, so there the tolerance mode runs the exact kernel and is checked
bit for bit.

At 176.4 and 192 kHz the fragment (fs / 20 = 8820 / 9600 frames) is longer than B200M_MAX_BLOCK, so a full block completes one
fragment edge or none: K1's chunk plan, the fragment kernels, the loudness log and the dBTP plane's split are run there in exact
mode against the reference, and the fused EBUr128 kernel in tolerance mode against an exact bank.
"""
import numpy as np
import pytest
from scipy.signal import lfilter, sosfilt

import _oracle as O
import _signals as S
from test_ebu_log_gpu import _Oracle as _LogOracle
from test_r128_fused_gpu import _Trio, R128F_MIN_CH
from test_r128_tplog_gpu import _TpOracle, _db

pytestmark = pytest.mark.gpu

RATES = (44100, 88200, 96000, 176400, 192000)
TOL_DB = 1e-4                        # true peak, K-meter, spectrum, dBTP: the contract's +-1e-4 dB
COR_TOL = 1e-5                       # correlation: a ratio in [-1, 1]
COR_F64_TOL = 2e-6                   # cor_scan_kernel against the float64 restatement (measured <= 6.5e-7 on an H100 up to the bound)
COR_SCAN_MAX_MEMORY = 21600          # csrc/cor.cu: above 1 / w2 = tcf * fs samples the tolerance mode runs the exact kernel


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def dbv(v):
    with np.errstate(divide="ignore"):
        return 20.0 * np.log10(np.asarray(v, np.float64))


def _schedule(cycle, total):
    """block lengths repeating `cycle` until `total` frames"""
    out, n = [], 0
    while n < total:
        for b in cycle:
            b = min(b, total - n)
            if b:
                out.append(b); n += b
    return out


# ---- a. correlation ---------------------------------------------------------------------------------------------------------
COR_SIGNALS = ("noise, correlation 0.6", "identical", "inverted", "997 Hz tones 1 rad apart", "60 dB fade",
               "programme, then digital silence")
COR_CYCLE = [1024] * 20 + [8192, 777, 1, 4095, 8192, 33]


def _cor_signal(fs, off, n, dur):
    """frames off .. off + n - 1 of the six test pairs (rows 2 p, 2 p + 1), dur seconds in all"""
    w = S.white(2, n, seed=91, block=off).astype(np.float64) / S.gain_ladder(2)[:, None]
    a, b = 0.5 * w[0], 0.5 * w[1]
    t = (off + np.arange(n)) / fs
    c = np.stack([a, 0.6 * a + 0.8 * b])
    tone = 0.5 * np.stack([np.sin(2 * np.pi * 997.0 * t), np.sin(2 * np.pi * 997.0 * t + 1.0)])
    fade = 10.0 ** (-60.0 * t / dur / 20.0)
    x = np.concatenate([c, np.stack([a, a]), np.stack([a, -a]), tone, c * fade, c * (t < dur / 2)])
    return np.ascontiguousarray(x, np.float32)


class _CorF64:
    """Stcorrdsp (stcorrdsp.cc:47-82) in float64 with the bank's float32 coefficients: zl, zr and the three product filters as
    one-pole filters, the end-of-process +1e-10 bias on the products at every block end (the scrub does nothing on finite input)"""

    def __init__(self, w, n):
        self.w1, self.w2 = float(w[0]), float(w[1])
        self.y = np.zeros((5, n))                          # zl zr zlr zll zrr

    def process(self, x, ends):
        """x [2n, m]: one stretch of blocks; ends: each block's end (exclusive) in x.  Returns the readings at the block ends."""
        a1, a2 = 1.0 - self.w1, 1.0 - self.w2
        x = x.astype(np.float64)
        zl = np.empty((2,) + x[0::2].shape)
        for k in range(2):
            zl[k], _ = lfilter([1.0], [1.0, -a1], self.w1 * x[k::2] + 1e-20, axis=1, zi=a1 * self.y[k][:, None])
        prods = (zl[0] * zl[1], zl[0] * zl[0], zl[1] * zl[1])
        bias = np.zeros(x.shape[1]); bias[np.asarray(ends) - 1] = 1e-10
        z = []
        for k, p in enumerate(prods):
            y, _ = lfilter([1.0], [1.0, -a2], self.w2 * p + bias, axis=1, zi=a2 * self.y[2 + k][:, None])
            z.append(y[:, np.asarray(ends) - 1])
        self.y[0], self.y[1] = zl[0][:, -1], zl[1][:, -1]
        for k in range(3):
            self.y[2 + k] = z[k][:, -1]
        return (z[0] / np.sqrt(z[1] * z[2] + 1e-10)).T      # [blocks, n]


def _cor_run(fs, dur, tcf=0.3):
    """a tolerance-mode bank fed plain blocks and the reference oracle over dur seconds; where the time-parallel kernel runs, also
    a bank fed ragged blocks, one attached to a phasewheel bank and the float64 restatement.  Returns the worst |reading - reference|
    and |reading - float64| per pair, the worst |reference - float64|, and whether the exact kernel ran."""
    import torch
    import meters_lv2_b200 as B
    n = len(COR_SIGNALS)
    plain, rag, att = (B.Stcorrdsp(n, fs, 2e3, tcf) for _ in range(3))
    for g in (plain, rag, att):
        g.set_precision(B.PREC_FMA)
    exact = plain.coeffs()[1] < np.float32(1) / np.float32(COR_SCAN_MAX_MEMORY)     # cor_launch's test, in float
    pw = B.Phasewheel(n, 1024, float(fs))
    pw.attach_cor(att)
    o = O.Stcorr(n, fs, 2e3, tcf)
    f = _CorF64(plain.coeffs(), n)
    pad = torch.full((2 * n, 8192), float("nan"), device="cuda")
    worst = {k: np.zeros(n) for k in ("ref", "f64", "ref_f64")}
    sched = _schedule(COR_CYCLE, int(dur * fs))
    cyc = sum(COR_CYCLE)
    for c0 in range(0, len(sched), len(COR_CYCLE)):
        blocks = sched[c0:c0 + len(COR_CYCLE)]
        off = c0 // len(COR_CYCLE) * cyc
        m = sum(blocks)
        x = _cor_signal(fs, off, m, dur)
        xd = torch.from_numpy(x).cuda()
        ends = np.cumsum(blocks)
        ref64 = None if exact else f.process(x, ends)
        a = 0
        for k, nb in enumerate(blocks):
            blk = xd[:, a:a + nb]
            plain.process(blk)
            if not exact:
                wide = min(nb + 7, 8192)                             # frames past each pair's length are NaN and must not count
                pad[:, :nb].copy_(blk); pad[:, nb:wide] = float("nan")
                rag.process(pad[:, :wide], lengths=[nb] * n)
                pw.process(blk)
            o.process(np.ascontiguousarray(x[:, a:a + nb]))
            a += nb
            g, r = plain.read().astype(np.float64), o.read().astype(np.float64)
            worst["ref"] = np.maximum(worst["ref"], np.abs(g - r))
            if exact:
                assert np.array_equal(u32(g), u32(r)), (fs, tcf, off + a)
                continue
            assert np.array_equal(u32(rag.read()), u32(g)), (fs, off + a)
            assert np.array_equal(u32(att.read()), u32(g)), (fs, off + a)
            worst["f64"] = np.maximum(worst["f64"], np.abs(g - ref64[k]))
            worst["ref_f64"] = np.maximum(worst["ref_f64"], np.abs(r - ref64[k]))
    return worst, exact


def _cor_report(tag, worst, exact):
    print("%s (%s kernel)" % (tag, "exact" if exact else "scan"))
    for i, s in enumerate(COR_SIGNALS):
        print("  %-32s vs reference %.3g" % (s, worst["ref"][i])
              + ("" if exact else "   vs float64 %.3g   reference vs float64 %.3g" % (worst["f64"][i], worst["ref_f64"][i])))


@pytest.mark.parametrize("fs", (44100, 48000, 88200, 96000, 176400, 192000))
def test_cor_tolerance_mode_at_rate(fs):
    """60 s of six pairs in 1024-frame blocks with odd and 8192-frame ones, read after every block.  Where the time-parallel
    kernel runs (44.1 and 48 kHz): every reading within COR_TOL of the reference and within COR_F64_TOL of float64 arithmetic, the
    ragged and the phasewheel-fed banks bit-identical to the plain one; above COR_SCAN_MAX_MEMORY (88.2-192 kHz) bit-identical to the
    reference"""
    worst, exact = _cor_run(fs, 60.0)
    _cor_report("%d Hz, tcf 0.3 s" % fs, worst, exact)
    assert exact == (0.3 * fs > COR_SCAN_MAX_MEMORY)
    if not exact:
        assert worst["f64"].max() <= COR_F64_TOL, worst["f64"]
    assert worst["ref"].max() <= COR_TOL, worst["ref"]


@pytest.mark.parametrize("tcf,exact", [(0.45, False), (1.0, True)])
def test_cor_tolerance_mode_time_constant(tcf, exact):
    """tcf is an argument: at 48 kHz 0.45 s is the longest memory the scan serves (21600 samples), 1 s is past it"""
    worst, ran_exact = _cor_run(48000, 20.0, tcf=tcf)
    _cor_report("48000 Hz, tcf %g s" % tcf, worst, ran_exact)
    assert ran_exact == exact
    if not exact:
        assert worst["f64"].max() <= COR_F64_TOL, worst["f64"]
    assert worst["ref"].max() <= COR_TOL, worst["ref"]


# ---- b. true peak / K-meter -------------------------------------------------------------------------------------------------
def _tpk_signal(C, fs, n, seed):
    x = S.white(C, n, seed=seed)
    t = np.arange(n) / fs
    x[1] = 0.9 * np.sin(2 * np.pi * 0.2371 * fs * t + 0.3)      # inter-sample peaks above the sample peaks
    x[2, n // 3:] = 0                                           # falls silent: hold expires, both filters decay
    x[3, :] = 0; x[3, 1000:1400] = 0.8                           # one burst, then silence
    x[4] *= 1e-4
    x[5] = 0
    x[6] = S.sine(n, 997.0, fs, amp=0.7)
    return np.ascontiguousarray(x, np.float32)


@pytest.mark.parametrize("fs", RATES)
@pytest.mark.parametrize("form", ["fused", "slabs"])
def test_tpk_kmeter_tolerance_mode_at_rate(fs, form, monkeypatch):
    """process() for 1.6 s (past the K-meter's 0.5 fs hold): true peak, its peak and the K-meter RMS within TOL_DB of the reference
    at every block, the K-meter peak bit-identical; an exact bank beside it stays bit-identical"""
    import torch
    import meters_lv2_b200 as B
    if form == "slabs":
        monkeypatch.setenv("B200M_TPK_SLAB", "256"); monkeypatch.setenv("B200M_TPK_SPLIT", "2")
    C = 37
    sizes = _schedule([1024] * 6 + [8192, 777, 4096, 3], int(1.6 * fs))
    n = sum(sizes)
    x = _tpk_signal(C, fs, n, seed=fs % 1009)
    g = B.TruePeakKmeter(C, float(fs)); g.set_precision(B.PREC_FMA)
    e = B.TruePeakKmeter(C, float(fs))
    ot = O.TruePeak(C, fs); ok = O.Kmeter(C, fs)
    xd = torch.from_numpy(x).cuda()
    a, worst = 0, 0.0
    for nb in sizes:
        blk = np.ascontiguousarray(x[:, a:a + nb])
        ot.process(blk, mode=0, nthreads=8); ok.process(blk, nthreads=8)
        g.process(xd[:, a:a + nb]); e.process(xd[:, a:a + nb])
        a += nb
        r, q = g.read(), e.read(); m, p = ot.read(); rms, pk = ok.read()
        assert np.array_equal(u32(q["tp_m"]), u32(m)) and np.array_equal(u32(q["tp_p"]), u32(p)), a
        assert np.array_equal(u32(q["km_rms"]), u32(rms)) and np.array_equal(u32(q["km_peak"]), u32(pk)), a
        assert np.array_equal(u32(r["km_peak"]), u32(pk)), a
        for got, ref in ((r["tp_m"], m), (r["tp_p"], p), (r["km_rms"], rms)):
            nz = ref > 1e-30
            assert np.all(np.abs(got[~nz] - ref[~nz]) <= 1e-30), a
            worst = max(worst, float(np.abs(dbv(got[nz]) - dbv(ref[nz])).max()))
    print("%d Hz %s: worst deviation %.3g dB" % (fs, form, worst))
    assert worst <= TOL_DB, worst


@pytest.mark.parametrize("fs", RATES)
def test_tpk_process_max_tensor_cores_at_rate(fs, monkeypatch):
    """process_max of a bank that gives every SM an 8-channel group (tpmax_tc_kernel), read every block, within TOL_DB"""
    import torch
    import meters_lv2_b200 as B
    monkeypatch.setenv("B200M_TPK_TC", "1")
    C = torch.cuda.get_device_properties(0).multi_processor_count * 8 + 5
    sizes = _schedule([1024, 8192, 512, 4096, 260], int(0.25 * fs))
    sizes = [s - s % 4 or 4 for s in sizes]
    n = sum(sizes)
    x = _tpk_signal(C, fs, n, seed=fs % 1013)
    g = B.TruePeakKmeter(C, float(fs), flags=B.TPK_TRUEPEAK); g.set_precision(B.PREC_FMA)
    ot = O.TruePeak(C, fs)
    xd = torch.from_numpy(x).cuda()
    a, worst = 0, 0.0
    for nb in sizes:
        ot.process(np.ascontiguousarray(x[:, a:a + nb]), mode=1, nthreads=8)
        g.process(xd[:, a:a + nb], tp_mode=1)
        a += nb
        r = g.read(); m, _ = ot.read()
        nz = m > 0
        assert np.array_equal(r["tp_m"][~nz], m[~nz]), a
        worst = max(worst, float(np.abs(dbv(r["tp_m"][nz]) - dbv(m[nz])).max()))
    print("%d Hz tensor cores: worst deviation %.3g dB" % (fs, worst))
    assert worst <= TOL_DB, worst


# ---- c. spectrum ------------------------------------------------------------------------------------------------------------
SPEC_Z_RTOL = 5e-8                   # biquad state vs the float64 restatement, relative to the instance's largest (measured <= 4.5e-9)


def _spec_band_centre(i):
    return 1000.0 * 2.0 ** ((i - 16) / 3.0)                 # spectrum_instantiate (spectrumlv2.c:73-121)


def _spec_signal(fs, n):
    """instance 0: tones at the centres of the five lowest bands (25-63 Hz); 1: a tone at the highest band's centre (below
    Nyquist) over noise; 2: noise, one channel 60 dB down"""
    t = np.arange(n) / fs
    low = sum(0.15 * np.sin(2 * np.pi * _spec_band_centre(i) * t + i) for i in range(5))
    top = min(_spec_band_centre(29), 0.45 * fs)
    w = S.white(4, n, seed=fs % 997)
    x = np.stack([low, low, 0.5 * np.sin(2 * np.pi * top * t) + 0.1 * w[0], 0.5 * np.sin(2 * np.pi * top * t + 1) + 0.1 * w[1],
                  w[2], 1e-3 * w[3]])
    return np.ascontiguousarray(x, np.float32)


def _spec_f64(W, x):
    """the band cascades (spectr.c:68-87) over a whole stereo stream in float64: input (l + r) / 2 in float, then the +-1e-12
    dither that alternates every sample; returns the final state [30, 6, 2]"""
    v = ((x[0] + x[1]) / np.float32(2)).astype(np.float64)
    v = v + np.where(np.arange(v.size) % 2 == 0, 1e-12, -1e-12)
    z = np.empty((30, 6, 2))
    for b in range(30):
        sos = np.array([[w[3], w[4], w[5], w[0], w[1], w[2]] for w in W[b]])
        _, z[b] = sosfilt(sos, v, zi=np.zeros((6, 2)))
    return z


@pytest.mark.parametrize("fs", RATES)
def test_spectrum_tolerance_mode_at_rate(fs):
    """2 s: levels and maxima within 1e-4 dB of the reference after every block, the fp64 biquad states within SPEC_Z_RTOL of
    the float64 restatement (and the exact bank's, bit-identical to the reference, too)"""
    import torch
    import meters_lv2_b200 as B
    n_inst = 3
    sizes = _schedule([1024] * 8 + [8192, 777, 1], int(2 * fs))
    n = sum(sizes)
    x = _spec_signal(fs, n)
    g = B.Spectr30(n_inst, 2, float(fs)); g.set_precision(B.PREC_FMA)
    o = O.Spectr30(n_inst, 2, float(fs))
    xd = torch.from_numpy(x).cuda()
    a, worst = 0, 0.0
    for nb in sizes:
        g.process(xd[:, a:a + nb]); o.process(np.ascontiguousarray(x[:, a:a + nb]), nthreads=3)
        a += nb
        gp, op = g.read().astype(np.float64), o.read().astype(np.float64)
        live = op > -100
        assert np.array_equal(live, gp > -100), a
        worst = max(worst, float(np.abs(gp[live] - op[live]).max()))
    W = g.coeffs()
    zdev = 0.0
    for inst in range(n_inst):
        z, _, _ = g.state(inst); oz, _, _ = o.state(inst)
        zf = _spec_f64(W, x[2 * inst:2 * inst + 2])
        scale = np.abs(zf).max()
        zdev = max(zdev, float(np.abs(z - zf).max() / scale))
        assert (np.abs(oz - zf) <= SPEC_Z_RTOL * scale).all(), inst
        assert (np.abs(z - zf) <= SPEC_Z_RTOL * scale).all(), (inst, float(np.abs(z - zf).max() / scale))
    print("%d Hz: worst port deviation %.3g dB, state vs float64 %.3g relative" % (fs, worst, zdev))
    assert worst <= TOL_DB, worst


# ---- d. EBUr128 where a fragment can be longer than a block -----------------------------------------------------------------
R128_SCHED = [8192, 8192, 1024, 8192, 4410, 8192, 7000, 1, 8192, 3, 8192, 9600 - 8192, 8192, 8192, 8192, 1024, 4800, 4800]
R128_FIELDS = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max",
               "range_thr")


def _r128_signal(nrows, off, nfram, fs):
    """a level that swings over some 40 dB at another rate on every instance, and one instance that is silent"""
    x = S.white(nrows, nfram, seed=17, block=off)
    t = (off + np.arange(nfram, dtype=np.float64)) / fs
    per = 1.5 + (np.arange(nrows) // 2 % 5)[:, None]
    env = 10.0 ** ((-25.0 + 20.0 * np.sin(2 * np.pi * t[None, :] / per)) / 20.0)
    x = x * env
    x[2:4] = 0
    return np.ascontiguousarray(x, np.float32)


@pytest.mark.parametrize("fs", (88200, 96000, 176400, 192000))
def test_r128_exact_and_log_at_rate(fs):
    """8 s in blocks of 8192 frames and blocks that straddle fragment edges, an exact bank with the loudness log and its dBTP
    plane: every EBU float, both histograms and the hold bit-identical to private reference instances, every log point too.  A
    tolerance-mode bank beside it logs the same loudness fields and dBTP points within TOL_DB"""
    import torch
    import meters_lv2_b200 as B
    n = 6
    fragm = fs // 20
    ex, tol = B.EBUr128(n, float(fs), True), B.EBUr128(n, float(fs), True)
    tol.set_precision(B.PREC_FMA)
    for bank in (ex, tol):
        bank.control(bank.START)
        bank.log_enable(512, dbtp=True)
    lo, to = _LogOracle(n, float(fs)), _TpOracle(n, 2, float(fs))
    lo.integr("start")
    sizes = _schedule(R128_SCHED, 8 * fs)
    a, none_edge, one_edge = 0, 0, 0
    for nb in sizes:
        x = _r128_signal(2 * n, a, nb, fs)
        e = (a + nb) // fragm - a // fragm
        none_edge += nb == 8192 and e == 0
        one_edge += nb == 8192 and e == 1
        a += nb
        xd = torch.from_numpy(x).cuda()
        ex.run(xd); tol.run(xd)
        lo.process(x); to.process(x)
    if fragm > 8192:
        assert none_edge and one_edge, (none_edge, one_edge)
    pe, ce, le = ex.log_drain(); pt, ct, lt = tol.log_drain()
    assert not le.any() and not lt.any()
    assert np.array_equal(ce, ct)
    re, tpe = ex.results(); rt, tpt = tol.results()
    assert re.tobytes() == rt.tobytes()
    worst = 0.0
    for i in range(n):
        ref = lo.e[i].read()[0]
        for k, name in enumerate(R128_FIELDS):
            assert u32(re[name][i]) == u32(ref[k]), (i, name)
        hm, hs = ex.histogram(i); om, os_, _ = lo.e[i].hist(0)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_), i
        pts = pe[i, :ce[i]]
        lp = lo.points(i)
        assert pts.shape[0] == lp.shape[0] == a // fragm, (i, pts.shape, lp.shape)
        for k, name in enumerate(("loudness_M", "loudness_S", "integrated", "range_min", "range_max")):
            assert np.array_equal(u32(pts[name]), u32(lp[:, k])), (i, name)
            assert np.array_equal(u32(pt[i, :ct[i]][name]), u32(lp[:, k])), (i, name)
        assert np.array_equal(u32(pts["dbtp"]), u32(to.points(i))), i
        hold = max(to.points(i).max(initial=-np.inf), _db(to.mx[i]))
        assert u32(tpe[i]) == u32(np.float32(hold)), (i, tpe[i], hold)
        dt, de = pt[i, :ct[i]]["dbtp"].astype(np.float64), pts["dbtp"].astype(np.float64)
        fin = np.isfinite(de)
        assert np.array_equal(fin, np.isfinite(dt)), i
        worst = max(worst, float(np.abs(dt[fin] - de[fin]).max(initial=0.0)), abs(float(tpt[i]) - float(tpe[i])) if fin.any() else 0.0)
    print("%d Hz: tolerance-mode dBTP points and hold within %.3g dB" % (fs, worst))
    assert worst <= TOL_DB, worst


@pytest.mark.parametrize("fs", (88200, 96000, 176400, 192000))
def test_r128_fused_kernel_at_rate(fs):
    """a tolerance-mode bank of R128F_MIN_CH channels runs r128_fused_kernel (K-weighting at this rate's coefficients and the
    tensor-core FIR in one kernel) on blocks of whole float4 rows: EBU floats and histograms bit-identical to an exact bank, the
    dBTP hold to the sliced host path, and within TOL_DB of the reference on a subset of instances"""
    import torch
    n_inst = R128F_MIN_CH // 2
    tri = _Trio(n_inst, fs=float(fs), n_ref=8)
    lvl = np.repeat(10.0 ** np.random.default_rng(fs).uniform(-3.5, 0.0, n_inst), 2).astype(np.float32)[:, None]
    lvl[::194] = 0.0                                           # some silent instances
    t0 = 0
    for i, nb in enumerate([8192, 8192, 1022, 8192, 4000, 8192, 8192]):
        x = S.white(2 * n_inst, nb, seed=fs % 1000, block=t0) * lvl; t0 += nb
        lf, le = tri.run(torch.from_numpy(x).cuda(), x)
        assert le - lf == (1 if nb % 4 == 0 else 0), (i, nb, lf, le)
        if i >= 2:
            tri.check((fs, i, nb))
