"""GPU: phasewheel / stereoscope FFT analysis bank.

The reference uses FFTW3 (gui/fft.c:234; not vendored, not installed, version unpinned), so this path is pinned to an
INDEPENDENT float64 FFT instead (numpy / pocketfft, tests/_fftref.py): test_fft_pinned_to_numpy_every_size checks Re / Im layout,
power and phase of b200m_pw_raw for every size the GUI offers, with the contract's tolerance (+-1e-4 dB, BASELINE.json north_star)
on every bin within 20 dB of the frame peak -- two fp32 transforms cannot agree better than ~3e-7 of the largest |X|, which
is 1e-4 dB at 20-25 dB below it -- and |dX| <= 1.5e-6 max|X| on all bins.  The process_audio logic around the transform (gates,
smoothing, peak) is compared with the CPU restatement, itself pinned to numpy by tests/test_oracle_port.py."""
import numpy as np
import pytest

import _oracle as O
import _signals as S

pytestmark = pytest.mark.gpu


def _compare(n_inst, bins, blocks, x, thr=1e-6):
    import torch
    import meters_lv2_b200 as B
    g = B.Phasewheel(n_inst, bins); o = O.Phasewheel(n_inst, bins, kind="port")
    g.debug_capture(True)
    xd = torch.from_numpy(x).cuda()
    pos = 0
    nfired = 0
    for n in blocks:
        fg = g.process(xd[:, pos:pos + n], thr); fo = o.process(np.ascontiguousarray(x[:, pos:pos + n]), thr, nthreads=8)
        assert fg == fo
        pos += n
        if fg:
            nfired += 1
            for inst in (0, n_inst - 1):
                gl, gr_, gpl, gpr = g.raw(inst); ol, or_, opl, opr = o.raw(inst)
                for a, b in ((gl, ol), (gr_, or_)):
                    scale = b.max()
                    # |X|^2 error for amplitude error eps*max|X| : <= 2*eps*sqrt(P*Pmax) + eps^2 Pmax
                    tol = 2 * 2e-6 * np.sqrt(np.maximum(b, 0) * scale) + 1e-11 * scale
                    assert (np.abs(a - b) <= tol + 1e-30).all(), float(np.abs(a - b).max() / scale)
            ph, lv, pk = g.read(); oph, olv, opk = o.read()
            live = (olv > -100) & (lv > -100)
            assert (live.sum() >= 0.98 * (olv > -100).sum())            # gate decisions agree except at the threshold
            d = np.angle(np.exp(1j * (ph - oph)))[live]
            strong = olv[live] > 1e-4 * olv.max()
            assert np.abs(d[strong]).max() < 2e-3 if strong.any() else True
            near = live & (olv >= 1e-2 * olv.max())                    # within 20 dB of the frame peak: the contract's 1e-4 dB = 2.3e-5 in power
            assert np.allclose(lv[near], olv[near], rtol=2.3e-5, atol=0)
            assert np.allclose(lv[live], olv[live], rtol=0, atol=3e-6 * float(olv.max()))
            assert np.allclose(pk, opk, rtol=2.3e-5, atol=1e-12)
    return nfired


def test_phasewheel_2048_white_noise():
    x = S.white(2 * 6, 1024 * 8, seed=41)
    assert _compare(6, 1024, [1024] * 8, x) == 4            # hop = 2 blocks (sps = 1920)


def test_phasewheel_tones_and_phase_difference():
    import torch
    import meters_lv2_b200 as B
    n = 1024 * 4
    f = 48000.0 * 100 / 2048                                  # bin-centred tone
    l = S.sine(n, f, amp=0.5); r = S.sine(n, f, amp=0.5, phase=np.pi / 3)
    x = np.ascontiguousarray(np.stack([l, r]))
    g = B.Phasewheel(1, 1024)
    xd = torch.from_numpy(x).cuda()
    for b in range(4):
        g.process(xd[:, b * 1024:(b + 1) * 1024])
    ph, lv, pk = g.read()
    assert abs(ph[0, 100] - np.pi / 3) < 1e-3 and lv[0, 100] > 1e-3


@pytest.mark.parametrize("bins", [64, 128, 256, 512, 1024, 2048, 4096, 6144, 8192])
def test_fft_pinned_to_numpy_every_size(bins):
    """every fft_bins value of the GUI's selector (gui/phasewheel.c:1108-1116) against numpy's float64 FFT"""
    import torch
    import meters_lv2_b200 as B
    import _fftref as F
    N = 2 * bins
    n_inst = 3
    total = max(3 * N, 6144)
    x = S.white(2 * n_inst, total, seed=47)
    x[3] = 0.5 * S.sine(total, 48000.0 * 37 / N, phase=0.7)            # bin-centred tone, known phase
    x[4] *= 1e-3                                                         # a quiet channel next to a loud one
    g = B.Phasewheel(n_inst, bins); g.debug_capture(True)
    xd = torch.from_numpy(x).cuda()
    pos, fired_end = 0, -1
    step = min(2048, N)                                                  # blocks no longer than the window: an analysis fires at a block end
    while pos + step <= total:
        if g.process(xd[:, pos:pos + step]):
            fired_end = pos + step
        pos += step
    assert fired_end >= N
    X, P, PH = F.spectra(x[:, fired_end - N:fired_end])
    worst = [0.0, 0.0, 0.0]
    for inst in range(n_inst):
        pl, pr, fl, fr = g.raw(inst)
        for ch, (pw, ph) in enumerate(((pl, fl), (pr, fr))):
            rel, db, dph = F.compare(pw, ph, X[2 * inst + ch])
            worst = [max(a, b) for a, b in zip(worst, (rel, db, dph))]
            x0 = X[2 * inst + ch][0].real                                                                         # power[0] = out[0]^2, phase[0] = 0
            assert abs(np.sqrt(float(pw[0])) - abs(x0)) <= 1.5e-6 * np.sqrt(P[2 * inst + ch].max()) and ph[0] == 0
            assert pw[bins - 1] == 0 and ph[bins - 1] == 0                                                        # never written (i < data_size - 1)
    print("fft_bins %5d N %5d: max|dX|/max|X| %.2e, bins within 20 dB of the peak: %.2e dB, %.2e rad" % (bins, N, *worst))
    assert worst[0] <= 1.5e-6 and worst[1] <= 1e-4 and worst[2] <= 5e-5, worst
    assert abs(g.raw(1)[3][37] - np.angle(X[3][37])) < 2e-5              # the tone's phase


@pytest.mark.parametrize("bins,blocks", [(64, [64] * 70), (256, [480] * 20), (4096, [8192] * 2 + [1000] * 3), (512, [1, 3, 1023, 4097, 777]), (6144, [8192, 5000, 8192, 1000])])
def test_other_sizes_and_ragged_blocks(bins, blocks):
    x = S.white(2 * 3, sum(blocks), seed=42)
    _compare(3, bins, blocks, x)


@pytest.mark.parametrize("bins", [512, 1024])
def test_stereoscope_process_audio(bins):
    """stereoscope mode (gui/stereoscope.c:705-741): smoothed lr[] / level[] after the same two FFTs; tolerance as for the
    phasewheel path (FFT "parity unpinned"), the smoothing itself is restated operation for operation"""
    import torch
    import meters_lv2_b200 as B
    n_inst, nb = 5, 24
    x = S.white(2 * n_inst, 1024 * nb, seed=43)
    x[1] *= 0.25; x[2] = x[3]                                   # hard-left-ish pair, identical pair (lr -> 0.5)
    x[4:6, 1024 * 10:] = 0.0                                    # goes silent: lr = 0.5, level = 0 branch
    g = B.Phasewheel(n_inst, bins); g.set_mode(1)
    o = O.Phasewheel(n_inst, bins, kind="port"); o.set_mode(1)
    xd = torch.from_numpy(x).cuda()
    fired = 0
    for b in range(nb):
        fg = g.process(xd[:, b * 1024:(b + 1) * 1024]); fo = o.process(np.ascontiguousarray(x[:, b * 1024:(b + 1) * 1024]), nthreads=4)
        assert fg == fo
        fired += fg
        lr, lv, _ = g.read(); olr, olv, _ = o.read()
        assert np.allclose(lv[:, 1:bins - 1], olv[:, 1:bins - 1], rtol=3e-4, atol=1e-9 * max(1e-30, float(olv.max())))
        strong = olv[:, 1:bins - 1] > 1e-5 * olv.max()
        assert np.abs(lr[:, 1:bins - 1] - olr[:, 1:bins - 1])[strong].max() < 2e-3 if strong.any() else True
    assert fired >= 10
    lr, lv, _ = g.read()
    assert abs(float(np.median(lr[1, 1:bins - 1])) - 0.5) < 0.02          # identical channels sit in the middle
    assert float(np.median(lr[0, 1:bins - 1])) < 0.35                     # right channel 12 dB down: pulled left
