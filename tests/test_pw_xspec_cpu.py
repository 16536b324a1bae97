"""CPU: the oracle of the phasewheel bank's cross-spectrum plane (tests/_pw_xspec.py) and the host-side parts of programme_stereo:
the band fields (stereo_bands), the window's noise bandwidth and the album pooling (stereo_albums).  No GPU."""
import numpy as np
import pytest

import _fftref as F
import _oracle as O
import _pw_xspec as X
import _signals as S

HAVE_PORT = O.available("port")


def _bands(sums, analyses, rate, bins):
    import meters_lv2_b200 as B
    return B.stereo_bands(sums, analyses, rate, bins)


def _pw_oracle_or_skip(n, bins, rate=48000.0):
    try:
        return O.Phasewheel(n, bins, rate, kind="port")
    except RuntimeError as e:
        pytest.skip(str(e))


@pytest.mark.skipif(not HAVE_PORT, reason="needs oracle/liboracle_port.so")
@pytest.mark.parametrize("bins,blocks", [(64, [64] * 70), (256, [480] * 20), (4096, [8192] * 2 + [1000] * 3), (512, [1, 3, 1023, 4097, 777]),
                                         (6144, [8192, 5000, 8192, 1000]), (64, [8192, 300, 8192]), (256, [8192, 1, 5000])])
@pytest.mark.parametrize("rate", [48000.0, 44100.0, 192000.0])
def test_clock_matches_the_restatement(bins, blocks, rate):
    """the oracle's firing clock reports an analysis in exactly the calls where the CPU restatement's fftx_run completes one, for the
    block patterns of the phasewheel tests and for blocks longer than the window (several analyses per call)"""
    o = _pw_oracle_or_skip(1, bins, rate)
    x = S.white(2, sum(blocks), seed=600)
    ends, fired = X.clock(blocks, bins, rate)
    pos, got = 0, []
    for n in blocks:
        got.append(o.process(np.ascontiguousarray(x[:, pos:pos + n])))
        pos += n
    assert got == fired
    sps = int(np.ceil(rate / 25))
    assert all(b - a >= sps for a, b in zip(ends, ends[1:]))      # the count restarts from 0 at each analysis
    if max(blocks) >= 2 * (sps + 2 * bins):
        assert len(ends) > sum(fired)                        # some call analysed more than once


def test_clock_steps():
    # N = 128, sps = 1920: a call of 8192 frames is 64 steps of 128; the clock fires at the 15th step (1920 frames) and every 15 after
    ends, fired = X.clock([8192], 64, 48000.0)
    assert ends == [1920, 3840, 5760, 7680] and fired == [1]
    ends, fired = X.clock([1000, 0, 1000, 1000], 1024, 48000.0)      # steps of min (2048, n): fires once the count reaches 1920
    assert ends == [2000] and fired == [0, 0, 1, 0]


def test_enbw_matches_the_reference_window():
    import meters_lv2_b200 as B
    for bins in (64, 512, 1024, 2048, 6144, 8192):
        w = F.hann_window(2 * bins).astype(np.float64)
        assert np.array_equal(B.pw_window(bins), F.hann_window(2 * bins))
        assert B.pw_enbw(bins) == w.size * float((w * w).sum()) / float(w.sum()) ** 2
        assert 1.5 < B.pw_enbw(bins) < 1.52


def test_band_membership_at_the_edges():
    import meters_lv2_b200 as B
    rate, bins = 48000.0, 1024
    df = rate / (2 * bins)
    lo, hi = B.SPEC_BAND_HZ * 2 ** (-1 / 6), B.SPEC_BAND_HZ * 2 ** (1 / 6)
    for b in (5, 16, 29):
        k0 = int(np.ceil(lo[b] / df))                        # the first bin at or above the band's lower edge
        inside, outside = np.zeros((1, 4, bins)), np.zeros((1, 4, bins))
        inside[0, :2, k0] = 1.0
        outside[0, :2, k0 - 1] = 1.0
        d = B.stereo_bands(inside, [1], rate, bins)
        assert np.isfinite(d["band_level_db"][0, b]).all()
        assert (k0 - 1) * df < lo[b] or (k0 - 1) * df >= hi[b - 1]
        d = B.stereo_bands(outside, [1], rate, bins)
        assert (d["band_level_db"][0, b] == -np.inf).all()
    # a bin exactly on an edge belongs to the band above: 48 kHz, 6144 bins (df = 3.90625 Hz): no band edge is a bin, so use a rate
    # that puts bin 256 exactly on band 16's lower edge
    bins = 1024
    rate = lo[16] / 256 * 2 * bins
    s = np.zeros((1, 4, bins)); s[0, :2, 256] = 1.0
    d = B.stereo_bands(s, [1], rate, bins)
    assert np.isfinite(d["band_level_db"][0, 16]).all() and (d["band_level_db"][0, 15] == -np.inf).all()


def test_empty_bands_dc_and_nan_rules():
    import meters_lv2_b200 as B
    rate, bins = 48000.0, 64                                 # 375 Hz bins: the low bands hold no bin
    s = np.zeros((3, 4, bins))
    s[0, 0] = 1.0; s[0, 1] = 1.0                             # L = R power, C = 0
    s[1, 0] = 1.0                                            # R silent
    s[:, :, 0] = 7.0                                         # DC is in no band
    d = B.stereo_bands(s, [1, 1, 0], rate, bins)
    band = B._stereo_band_of_bin(rate, bins)
    empty = np.bincount(band[band >= 0], minlength=30) == 0
    assert empty[:10].all() and not empty[-5:].any()
    for f in ("band_corr", "band_coherence", "band_phase", "band_balance_db", "band_mono_db"):
        assert np.isnan(d[f][:, empty]).all(), f
    assert np.isnan(d["band_level_db"][:, empty]).all()
    live = ~empty
    assert (d["band_corr"][0, live] == 0).all() and (d["band_coherence"][0, live] == 0).all()
    assert np.isnan(d["band_phase"][0, live]).all()          # C is 0: no phase
    assert np.allclose(d["band_mono_db"][0, live], 10 * np.log10(0.5))
    assert (d["band_balance_db"][1, live] == -np.inf).all()  # RR = 0 over LL > 0
    assert (d["band_level_db"][1, live, 1] == -np.inf).all() and np.isnan(d["band_corr"][1, live]).all()
    assert np.isnan(d["band_level_db"][2]).all()             # no analysis: the level's denominator is 0
    # exact anti-phase: the downmix's power is 0
    a = np.zeros((1, 4, bins)); a[0, 0] = a[0, 1] = 2.0; a[0, 2] = -2.0
    d = B.stereo_bands(a, [1], rate, bins)
    assert (d["band_mono_db"][0, live] == -np.inf).all() and (d["band_corr"][0, live] == -1).all()


def test_level_scale():
    """a bin-centred sine of amplitude a reads 20 log10 a in its band: enbw turns the windowed lobe's power sum into a^2"""
    import meters_lv2_b200 as B
    rate, bins = 48000.0, 1024
    k = 43                                                   # 1007.8 Hz, band 16 (891 .. 1122 Hz)
    t = np.arange(6 * 2048)
    x = np.stack([0.5 * np.sin(2 * np.pi * k * t / 2048), 0.25 * np.sin(2 * np.pi * k * t / 2048)]).astype(np.float32)
    ends = [4096, 6144, 8192]
    r = X.analyse(x, ends, bins)
    d = B.stereo_bands(r["sums"][None], [r["analyses"]], rate, bins)
    assert abs(d["band_level_db"][0, 16, 0] - 20 * np.log10(0.5)) < 1e-3
    assert abs(d["band_level_db"][0, 16, 1] - 20 * np.log10(0.25)) < 1e-3
    assert abs(d["band_balance_db"][0, 16] - 20 * np.log10(0.5)) < 1e-6


@pytest.mark.parametrize("kind", ["same", "inverted", "half", "independent", "delay3"])
def test_known_answers_on_the_oracle(kind):
    rate, bins = 48000.0, 1024
    T = 48000 * 3
    x = np.empty((2, T), np.float32)
    x[0] = S.white(1, T, seed=610)[0]
    if kind == "same":
        x[1] = x[0]
    elif kind == "inverted":
        x[1] = -x[0]
    elif kind == "half":
        x[1] = x[0] * np.float32(0.5)
    elif kind == "independent":
        x[1] = S.white(1, T, seed=611)[0]
    else:
        x[1, 3:] = x[0, :-3]; x[1, :3] = 0
    ends, _ = X.clock([1024] * (T // 1024), bins, rate)
    r = X.analyse(x, ends, bins)
    s = r["sums"]
    assert r["analyses"] == len(ends) and r["skipped"] == 0
    d = _bands(s[None], [r["analyses"]], rate, bins)
    live = np.isfinite(d["band_corr"][0])
    if kind == "same":
        assert np.array_equal(s[0], s[1]) and np.array_equal(s[2], s[0]) and (s[3] == 0).all()
        assert np.allclose(d["band_corr"][0, live], 1.0) and np.allclose(d["band_mono_db"][0, live], 0.0, atol=1e-9)
    elif kind == "inverted":
        assert np.array_equal(s[2], -s[0]) and (d["band_mono_db"][0, live] < -200).all()
        assert np.allclose(d["band_corr"][0, live], -1.0)
    elif kind == "half":
        assert np.allclose(s[1], 0.25 * s[0], rtol=1e-12, atol=0) and np.allclose(s[2], 0.5 * s[0], rtol=1e-12, atol=0)
        assert np.allclose(d["band_balance_db"][0, live], 20 * np.log10(0.5), atol=1e-9)
    elif kind == "independent":
        hi = B_above(250.0) & live
        assert np.abs(d["band_mono_db"][0, hi] + 3.0103).max() < 0.5
        assert np.abs(d["band_corr"][0, B_above(1000.0) & live]).max() < 0.1
    else:
        k = np.arange(bins)
        strong = s[0] > 1e-2 * s[0].max()
        strong[0] = False
        ph = np.arctan2(s[3], s[2])
        want = -2 * np.pi * (k * rate / (2 * bins)) * 3 / rate
        assert np.abs(np.angle(np.exp(1j * (ph - want))))[strong].max() < 0.02


def B_above(hz):
    import meters_lv2_b200 as B
    return B.SPEC_BAND_HZ * 2 ** (-1 / 6) >= hz


def _rows(n, bins, seed):
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((n, 4, bins)) * np.exp(rng.standard_normal((n, 1, 1)) * 10)
    s[:, :2] = np.abs(s[:, :2])
    return s, rng.integers(0, 50, n).astype(np.int64), rng.integers(0, 3, n).astype(np.int64)


def test_albums_pool_in_clip_order():
    import meters_lv2_b200 as B
    rate, bins = 48000.0, 256
    s, a, k = _rows(9, bins, 620)
    grp = np.array([2, 0, -1, 2, 0, 2, 4, -1, 0])
    d = B.stereo_albums(s, a, k, grp, rate, bins)
    assert d["album_sums"].shape == (5, 4, bins)
    want = np.zeros((5, 4, bins))
    for i in range(9):                                       # ascending clip index
        if grp[i] >= 0:
            want[grp[i]] += s[i]
    assert np.array_equal(d["album_sums"].view(np.uint64), want.view(np.uint64))
    assert list(d["album_n_clips"]) == [3, 0, 3, 0, 1]
    assert list(d["album_analyses"]) == [a[[1, 4, 8]].sum(), 0, a[[0, 3, 5]].sum(), 0, a[6]]
    assert list(d["album_skipped"]) == [k[[1, 4, 8]].sum(), 0, k[[0, 3, 5]].sum(), 0, k[6]]
    assert (d["album_sums"][[1, 3]] == 0).all() and np.isnan(d["album_band_level_db"][[1, 3]]).all()
    ref = B.stereo_bands(want, d["album_analyses"], rate, bins)
    for f, v in ref.items():
        assert np.array_equal(d["album_" + f], v, equal_nan=True), f
    # two halves of the clips (two shards' rows gathered in clip order) pool to the same bits as one set of rows
    h1 = B.stereo_albums(s[:4], a[:4], k[:4], grp[:4], rate, bins)
    cat = [np.concatenate(v) for v in ((s[:4], s[4:]), (a[:4], a[4:]), (k[:4], k[4:]))]
    d2 = B.stereo_albums(*cat, grp, rate, bins)
    for f in d:
        assert np.array_equal(np.asarray(d[f]), np.asarray(d2[f]), equal_nan=True), f
    assert h1["album_sums"].shape[0] == 3
    none = B.stereo_albums(s[:2], a[:2], k[:2], [-1, -1], rate, bins)
    assert none["album_sums"].shape == (0, 4, bins) and none["album_n_clips"].shape == (0,)


def test_albums_and_bands_reject_bad_rows():
    import meters_lv2_b200 as B
    s, a, k = _rows(3, 64, 630)
    with pytest.raises(B.B200MError):
        B.stereo_bands(s, a[:2], 48000.0, 64)
    with pytest.raises(B.B200MError):
        B.stereo_bands(s, a, 48000.0, 128)
    with pytest.raises(B.B200MError):
        B.stereo_albums(s, a, k[:1], [0, 0, 0], 48000.0, 64)
    with pytest.raises(B.B200MError):
        B.stereo_albums(s, a, k, [0, 0], 48000.0, 64)
    with pytest.raises(B.B200MError):
        B.stereo_albums(s, a, k, [0, -2, 0], 48000.0, 64)
