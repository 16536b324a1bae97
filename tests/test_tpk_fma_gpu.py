"""GPU parity of the tolerance mode of the true-peak FIR (B200M_PREC_FMA, include/b200meters.h).

north_star: float outputs within +-1e-4 dB of the reference, integer results bit-exact.  The FMA mode changes the
4x polyphase FIR (zita-resampler/resampler.cc:213-230) and, in the fused process() kernel, the attack filters of the true-peak
ballistics (truepeakdsp.cc:57-84) and the K-meter's RMS filters (kmeterdsp.cc:80-97); the tolerance is written below as TOL_DB and checked on
 * the raw 4x stream against zita-resampler's own output (relative to the block peak, which is what a peak meter reads),
 * TruePeakdsp::process_max / process readings (jmeters/truepeakdsp.cc:41-124) in dB,
 * the EBUr128 cycle: dBTP hold within TOL_DB while every EBU float AND both histograms stay bit-identical.
"""
import numpy as np
import pytest

import _oracle as O
import _signals as S

pytestmark = pytest.mark.gpu

TOL_DB = 1e-4                      # the contract's tolerance (BASELINE.json north_star)
TOL_REL = 10 ** (TOL_DB / 20) - 1  # = 1.15e-5 relative on a linear reading


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def db(v):
    with np.errstate(divide="ignore"):
        return 20.0 * np.log10(np.asarray(v, np.float64))


@pytest.mark.parametrize("n,block", [(4096, 1024), (3000, 1000), (777, 777), (8192, 8192)])
def test_fma_stream_within_tolerance(n, block):
    import torch
    import meters_lv2_b200 as B
    x = S.white(9, n, seed=15)
    x[3] *= 1e-6; x[4] = 0
    x[5] = S.sine(n, 997.0, amp=0.9); x[6] = S.sine(n, 11025.0, amp=1.0, phase=np.pi / 4)    # inter-sample peaks
    g = B.TruePeakKmeter(9); g.set_precision(B.PREC_FMA); g.debug_capture(True)
    xd = torch.from_numpy(x).cuda()
    chans = (0, 3, 4, 5, 6, 8)
    outs = {ch: [] for ch in chans}
    for o in range(0, n, block):
        k = min(block, n - o)
        g.process(xd[:, o:o + k])
        for ch in chans:
            outs[ch].append(g.debug_upsampled(ch, 4 * k))
    for ch in chans:
        ref = O.tp_upsample(x[ch], block=block).astype(np.float64)
        got = np.concatenate(outs[ch]).astype(np.float64)
        peak = np.abs(ref).max()
        if peak == 0:
            assert np.all(got == 0)
            continue
        err = np.abs(got - ref).max() / peak
        assert err <= 0.2 * TOL_REL, (ch, err)                 # measured ~2e-7; the bound leaves 5x margin to the contract


@pytest.fixture(autouse=True, params=["default", "slabs"])
def process_form(request, monkeypatch):
    """process() runs fused for small banks; "slabs" forces the FIR / ballistics slab pipeline that large banks use"""
    if request.param == "slabs":
        monkeypatch.setenv("B200M_TPK_SLAB", "256"); monkeypatch.setenv("B200M_TPK_SPLIT", "2")
    return request.param


@pytest.mark.parametrize("mode", [0, 1])
def test_fma_readings_within_tolerance(mode):
    """process_max (mode 1) and process (mode 0) readings, 40 blocks of 1024, read every block"""
    import torch
    import meters_lv2_b200 as B
    C = 70
    x = S.white(C, 40 * 1024, seed=23)
    x[7] = S.sine(40 * 1024, 5512.5, amp=0.7, phase=0.3)
    g = B.TruePeakKmeter(C); g.set_precision(B.PREC_FMA)
    ot = O.TruePeak(C); ok = O.Kmeter(C)
    xd = torch.from_numpy(x).cuda()
    worst = 0.0
    for b in range(40):
        blk = np.ascontiguousarray(x[:, b * 1024:(b + 1) * 1024])
        ot.process(blk, mode=mode, nthreads=8); ok.process(blk, nthreads=8)
        g.process(xd[:, b * 1024:(b + 1) * 1024], tp_mode=mode)
        r = g.read(); m, p = ot.read(); rms, pk = ok.read()
        # the K-meter's peak is a maximum of squares: exact in either mode; its two RMS filters contract mul + add in the fused
        # process() kernel of the tolerance mode (the slab pipeline and process_max banks keep the exact ballistics)
        assert np.array_equal(u32(r["km_peak"]), u32(pk))
        for got, ref in ((r["tp_m"], m), (r["km_rms"], rms)) + (((r["tp_p"], p),) if mode == 0 else ()):
            nz = ref > 0
            assert np.array_equal(got[~nz], ref[~nz])
            d = np.abs(db(got[nz]) - db(ref[nz])).max()
            worst = max(worst, d)
    assert worst <= TOL_DB, worst
    print("worst deviation %.3g dB" % worst)
    assert worst <= 5e-5, "measured <= 1e-5 dB on this input: something regressed (%g)" % worst


def test_fma_r128_cycle_histograms_stay_bit_exact():
    """EBUr128 cycle with the dBTP FIR in tolerance mode: the nine EBU floats and both histograms are bit-identical to the
    reference, tp_max within TOL_DB."""
    import torch
    import meters_lv2_b200 as B
    n_inst, nb = 96, 135
    x = S.white(2 * n_inst, nb * 1024, seed=31)
    g = B.EBUr128(n_inst, 48000.0, True); g.set_precision(B.PREC_FMA); g.control(B.EBUr128.START)
    xd = torch.from_numpy(x).cuda()
    for b in range(nb):
        g.run(xd[:, b * 1024:(b + 1) * 1024])
    res, tp = g.results()
    oe = O.Ebu(n_inst, 2); ot = O.TruePeak(2 * n_inst); oe.integr("start")
    tpmax = np.full(n_inst, -np.inf, np.float32)
    for b in range(nb):
        blk = np.ascontiguousarray(x[:, b * 1024:(b + 1) * 1024])
        oe.process(blk, nthreads=8); ot.process(blk, mode=1, nthreads=8)
        m, _ = ot.read()
        v = np.maximum(m[0::2], m[1::2])
        with np.errstate(divide="ignore"):
            t = np.where(v == 0, -np.inf, (20.0 * np.log10(v.astype(np.float32)).astype(np.float64)).astype(np.float32))
        tpmax = np.maximum(tpmax, t)
    orr = oe.read()
    for i, k in enumerate(("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")):
        assert np.array_equal(u32(res[k]), u32(orr[:, i])), k
    for inst in (0, 17, n_inst - 1):
        hm, hs = g.ebu.histogram(inst); om, os_, _ = oe.hist(inst)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_)
    assert np.abs(tp.astype(np.float64) - tpmax.astype(np.float64)).max() <= TOL_DB


@pytest.mark.parametrize("km", [True, False])
def test_fma_process_ragged_blocks(km, process_form):
    """process() of a tolerance-mode bank (decoupled-role kernel, csrc/tpk.cu tpdec_kernel) over block lengths that are not multiples
    of its 24-sample chunks or of 4, from unaligned block starts, on a channel count that leaves a partial CTA"""
    import torch
    import meters_lv2_b200 as B
    C = 37
    sizes = [1, 3, 24, 25, 47, 48, 49, 95, 96, 97, 1000, 4096, 2, 8191, 1024, 5, 120]
    total = sum(sizes)
    x = S.white(C, total, seed=5)
    x[2] = S.sine(total, 997.0, amp=0.9, phase=0.1)
    x[5] = 0
    x[6, 3000:] = 0                                        # a channel that falls silent: the filters decay
    g = B.TruePeakKmeter(C, flags=(B.TPK_TRUEPEAK | B.TPK_KMETER) if km else B.TPK_TRUEPEAK)
    g.set_precision(B.PREC_FMA)
    ot = O.TruePeak(C); ok = O.Kmeter(C)
    xd = torch.from_numpy(x).cuda()
    a = 0; worst = 0.0
    for n in sizes:
        blk = np.ascontiguousarray(x[:, a:a + n])
        ot.process(blk, mode=0, nthreads=4); ok.process(blk, nthreads=4)
        g.process(xd[:, a:a + n], tp_mode=0)
        a += n
        r = g.read(); m, p = ot.read(); rms, pk = ok.read()
        pairs = [(r["tp_m"], m), (r["tp_p"], p)]
        if km:
            assert np.array_equal(u32(r["km_peak"]), u32(pk)), n
            pairs.append((r["km_rms"], rms))
        for got, ref in pairs:
            nz = ref > 1e-30
            assert np.all(np.abs(got[~nz] - ref[~nz]) <= 1e-30), n
            if nz.any():
                worst = max(worst, np.abs(db(got[nz]) - db(ref[nz])).max())
    print("worst deviation %.3g dB" % worst)
    assert worst <= TOL_DB, worst


def test_fma_process_max_tensor_core_path(monkeypatch):
    """process_max of a bank large enough for the tensor-core kernel (csrc/tpk.cu tpmax_tc_kernel: every SM gets an 8-channel group),
    over block lengths with partial tiles, a channel count that leaves a partial group, silent and constant channels, read every block"""
    import torch
    import meters_lv2_b200 as B
    monkeypatch.setenv("B200M_TPK_TC", "1")
    C = torch.cuda.get_device_properties(0).multi_processor_count * 8 + 21
    sizes = [1024, 1000, 512, 260, 4, 2048, 1024]
    total = sum(sizes)
    x = S.white(C, total, seed=11)
    x[3] = S.sine(total, 11025.0, amp=0.8, phase=0.4)       # inter-sample peaks above the sample peaks
    x[5] = 0
    x[9] = 0.25
    x[C - 1] *= 1e-5
    g = B.TruePeakKmeter(C, flags=B.TPK_TRUEPEAK); g.set_precision(B.PREC_FMA)
    ot = O.TruePeak(C)
    xd = torch.from_numpy(x).cuda()
    a = 0; worst = 0.0
    for n in sizes:
        blk = np.ascontiguousarray(x[:, a:a + n])
        ot.process(blk, mode=1, nthreads=8)
        g.process(xd[:, a:a + n], tp_mode=1)
        a += n
        r = g.read(); m, _ = ot.read()
        nz = m > 0
        assert np.array_equal(r["tp_m"][~nz], m[~nz]), n
        worst = max(worst, np.abs(db(r["tp_m"][nz]) - db(m[nz])).max())
    print("worst deviation %.3g dB" % worst)
    assert worst <= TOL_DB, worst
    assert worst <= 3e-5, worst
