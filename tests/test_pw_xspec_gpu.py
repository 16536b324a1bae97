"""GPU: the phasewheel bank's cross-spectrum plane (b200m_pw_xspec_enable / _read) and programme_stereo.

The bank's fp32 transform is pinned to numpy's float64 FFT (test_pw_gpu.py), so the plane is checked against the float64 oracle
tests/_pw_xspec.py within the bound it propagates from that pin, with the analysis counts exact.  Everything the plane must not change
(ports, peak, raw spectra, stereoscope smoothing, an attached correlation bank) and every path that must give the same rows (ragged
against private banks, lock step against ragged, host against device, fused against unfused) is compared bit for bit."""
import numpy as np
import pytest

import _pw_xspec as X
import _signals as S

pytestmark = pytest.mark.gpu

U64 = lambda a: np.ascontiguousarray(a, np.float64).view(np.uint64)


def _signal(n, T, seed):
    """n stereo pairs of T frames: noise, a tone pair and partly correlated channels"""
    x = S.white(2 * n, T, seed=seed)
    t = np.arange(T)
    x[0] = (0.3 * np.sin(2 * np.pi * 0.01731 * t) + 0.1 * x[0]).astype(np.float32)
    x[1] = (0.2 * np.sin(2 * np.pi * 0.01731 * t + 0.7) + 0.1 * x[1]).astype(np.float32)
    if n > 1:
        x[3] = (0.6 * x[2] + 0.4 * x[3]).astype(np.float32)
    return x


def _feed(g, x, blocks, lengths=None, **kw):
    import torch
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for j, nb in enumerate(blocks):
        if lengths is None:
            g.process(xd[:, pos:pos + nb], **kw)
        else:
            g.process(xd[:, pos:pos + nb], lengths=lengths[j], **kw)
        pos += nb
    return pos


BLOCKS = {"short": lambda bins: [1024] * 12 + [1, 777],
          "long": lambda bins: [8192, 5000, 8192, 3, 8192]}
CASES = [(b, 48000.0) for b in (64, 128, 256, 512, 1024, 2048, 4096, 6144, 8192)] + \
        [(b, r) for r in (44100.0, 96000.0, 192000.0) for b in (256, 4096)]


@pytest.mark.parametrize("bins,rate", CASES)
@pytest.mark.parametrize("blocks", ["short", "long"])
def test_plane_against_the_oracle(bins, rate, blocks):
    import meters_lv2_b200 as B
    n = 3
    bl = BLOCKS[blocks](bins)
    x = _signal(n, sum(bl), seed=700 + bins)
    g = B.Phasewheel(n, bins, rate)
    g.xspec_enable()
    _feed(g, x, bl)
    s, a, k = g.xspec()
    os_, ob, oa, ok = X.bank(x, [[nb] * n for nb in bl], bins, rate)
    assert np.array_equal(a, oa) and (k == 0).all() and (ok == 0).all()
    assert (oa > 0).all()
    err = np.abs(s - os_)
    assert (err <= ob).all(), float((err / np.maximum(ob, 1e-300)).max())
    # band values on the bands within 20 dB of the clip's strongest band
    d, od = B.stereo_bands(s, a, rate, bins), B.stereo_bands(os_, oa, rate, bins)
    lv = od["band_level_db"].max(axis=-1)
    strong = np.isfinite(lv) & (lv >= np.nanmax(np.where(np.isfinite(lv), lv, -np.inf), axis=1, keepdims=True) - 20)
    for f, tol in (("band_mono_db", 1e-4), ("band_corr", 1e-4), ("band_coherence", 1e-4)):
        e = np.abs(d[f] - od[f])[strong]
        assert e.max() <= tol, (f, float(e.max()))
    e = np.abs(d["band_level_db"] - od["band_level_db"])[strong]
    assert e.max() <= 1e-4, float(e.max())


def _pair(n, bins, mode, fused, capture=True):
    import meters_lv2_b200 as B
    banks = []
    for plane in (False, True):
        g = B.Phasewheel(n, bins)
        if mode:
            g.set_mode(mode)
        if capture:
            g.debug_capture(True)
        c = None
        if fused:
            c = B.Stcorrdsp(n)
            g.attach_cor(c)
        if plane:
            g.xspec_enable()
        banks.append((g, c))
    return banks


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("ragged", [False, True])
def test_ports_unchanged_by_the_plane(mode, fused, ragged):
    """phase, level, peak and raw after every block, and an attached correlation bank's readings and state, are bit-identical with
    the plane on or off; blocks longer than the window run plane-only analyses in between"""
    import torch
    n, bins = 4, 256
    bl = [1024, 8192, 300, 4097, 1, 2048, 8192]
    x = _signal(n, sum(bl), seed=710)
    e = X.clock(bl, bins, 48000.0)[0][4]
    x[4, e - 100:e - 90] = np.nan                               # instance 2: a non-finite spectrum (plain blocks)
    xd = torch.from_numpy(x).cuda()
    rng = np.random.default_rng(711)
    (g0, c0), (g1, c1) = _pair(n, bins, mode, fused)
    pos = 0
    for nb in bl:
        ln = rng.integers(0, nb + 1, n) if ragged else None
        if ragged:
            ln[0] = nb
        f0 = g0.process(xd[:, pos:pos + nb], lengths=ln); f1 = g1.process(xd[:, pos:pos + nb], lengths=ln)
        assert f0 == f1
        pos += nb
        for u, v in zip(g0.read(), g1.read()):
            assert np.array_equal(u.view(np.uint32), v.view(np.uint32))
        for i in range(n):
            for u, v in zip(g0.raw(i), g1.raw(i)):
                assert np.array_equal(u.view(np.uint32), v.view(np.uint32))
        if fused:
            assert np.array_equal(c0.read().view(np.uint32), c1.read().view(np.uint32))
            for u, v in zip(c0.state(), c1.state()):
                assert np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8))
    s, a, k = g1.xspec()
    assert a.sum() > 0 and (ragged or k[2] > 0)


def test_rows_ragged_against_private_banks_and_paths():
    """a ragged bank of clips of different lengths (0 and 1 frame included) gives each clip the row of a private one-instance bank
    fed only that clip; lock step equals ragged with equal lengths; the host path on the bank's stream equals the device path on a
    caller stream; the fused correlation feed equals the unfused one"""
    import torch
    import meters_lv2_b200 as B
    n, bins, rate = 6, 128, 48000.0
    lens = np.array([0, 1, 3000, 20000, 41000, 41000])
    block = 4096
    nblk = -(-int(lens.max()) // block)
    x = _signal(n, nblk * block, seed=720)
    calls = [np.clip(lens - b * block, 0, block) for b in range(nblk)]
    g = B.Phasewheel(n, bins, rate); g.xspec_enable()
    _feed(g, x, [block] * nblk, calls)
    s, a, k = g.xspec()
    for i in range(n):
        p = B.Phasewheel(1, bins, rate); p.xspec_enable()
        if lens[i]:
            _feed(p, np.ascontiguousarray(x[2 * i:2 * i + 2, :lens[i]]), [min(block, lens[i] - o) for o in range(0, lens[i], block)])
        ps, pa, pk = p.xspec()
        assert np.array_equal(U64(ps[0]), U64(s[i])) and pa[0] == a[i] and pk[0] == k[i], i
        p.close()
    assert a[0] == 0 and a[1] == 0 and (s[:2] == 0).all() and a[-1] > 10
    os_, ob, oa, _ = X.bank(x, calls, bins, rate)
    assert np.array_equal(a, oa) and (np.abs(s - os_) <= ob).all()

    # lock step against ragged with equal lengths, host against device on a caller stream, fused against unfused
    bl = [1024, 8192, 777, 8192]
    y = _signal(n, sum(bl), seed=721)
    rows = {}
    yr = np.concatenate([y, y[:2]])
    for form in ("lock", "ragged", "host", "fused"):
        h = B.Phasewheel(n + (form == "ragged"), bins, rate)
        c = None
        if form == "fused":
            c = B.Stcorrdsp(n); h.attach_cor(c)
        h.xspec_enable()
        pos = 0
        st = torch.cuda.Stream()
        for nb in bl:
            if form == "host":
                h.process(np.ascontiguousarray(y[:, pos:pos + nb]))
            elif form == "ragged":                                # an extra instance of other lengths keeps the bank on the ragged path
                h.process(torch.from_numpy(yr[:, pos:pos + nb]).cuda(), lengths=np.r_[np.full(n, nb), nb // 2])
            elif form == "lock":
                yd = torch.from_numpy(y[:, pos:pos + nb]).cuda()
                torch.cuda.synchronize()
                with torch.cuda.stream(st):
                    h.process(yd, stream=st)
            else:
                h.process(torch.from_numpy(y[:, pos:pos + nb]).cuda())
            pos += nb
        rows[form] = [r[:n] for r in h.xspec(stream=st if form == "lock" else None)]
        h.close()
        if c is not None:
            c.close()
    for form in ("ragged", "host", "fused"):
        for u, v in zip(rows["lock"], rows[form]):
            assert np.array_equal(np.asarray(u).view(np.uint64), np.asarray(v).view(np.uint64)), form


def test_non_finite_and_denormal_input():
    import meters_lv2_b200 as B
    n, bins, rate = 3, 256, 48000.0
    bl = [1024] * 30
    x = _signal(n, sum(bl), seed=730)
    clean = x.copy()
    ends = X.clock(bl, bins, rate)[0]                           # every 2048 frames: N = 512 < sps, so a sample is in one window at most
    x[2, ends[2] - 10] = np.nan                                 # instance 1, L
    x[3, ends[5] - 100] = np.inf                                # instance 1, R
    x[4:6] = (x[4:6] * np.float32(1e-39)).astype(np.float32)    # instance 2: denormal input
    clean[4:6] = x[4:6]
    g = B.Phasewheel(n, bins, rate); g.xspec_enable()
    _feed(g, x, bl)
    s, a, k = g.xspec()
    h = B.Phasewheel(n, bins, rate); h.xspec_enable()
    _feed(h, clean, bl)
    cs, ca, ck = h.xspec()
    os_, ob, oa, ok = X.bank(x, [[nb] * n for nb in bl], bins, rate)
    assert np.array_equal(a, oa) and np.array_equal(k, ok)
    assert k[1] == 2 and k[0] == 0 and k[2] == 0 and a[2] == ca[2] > 0
    assert a[1] + k[1] == ca[1] and a[1] > 6                    # it accumulates again once the ring has flushed
    for i in (0, 2):                                            # the other instances are unaffected
        assert np.array_equal(U64(s[i]), U64(cs[i]))
    # subnormal fp32 values carry fewer significant bits, so the FFT pin's relative bound holds for the normal instances only
    assert np.isfinite(s).all() and (np.abs(s[:2] - os_[:2]) <= ob[:2]).all()
    assert (s[2, :2] > 0).any()                                 # denormal input adds like any other


def test_enable_disable_reenable():
    import meters_lv2_b200 as B
    n, bins = 2, 512
    x = _signal(n, 1024 * 20, seed=740)
    g = B.Phasewheel(n, bins)
    with pytest.raises(B.B200MError):
        g.xspec()
    _feed(g, x[:, :4096], [1024] * 4)
    g.xspec_enable()
    s, a, k = g.xspec()
    assert (s == 0).all() and (a == 0).all() and (k == 0).all()
    _feed(g, np.ascontiguousarray(x[:, 4096:8192]), [1024] * 4)
    s1, a1, _ = g.xspec()
    assert (a1 == 2).all()                                      # sps = 1920: positions 5760 and 7680
    g.xspec_enable(False)
    _feed(g, np.ascontiguousarray(x[:, 8192:12288]), [1024] * 4)
    s2, a2, _ = g.xspec()
    assert np.array_equal(U64(s1), U64(s2)) and np.array_equal(a1, a2)   # off: nothing added, rows kept
    g.set_mode(1); g.debug_capture(True)                         # neither touches the plane
    assert np.array_equal(U64(g.xspec()[0]), U64(s1))
    g.xspec_enable()
    assert (g.xspec()[0] == 0).all() and (g.xspec()[1] == 0).all()   # enabling zeroes, also when the memory is there
    _feed(g, np.ascontiguousarray(x[:, 12288:16384]), [1024] * 4)
    assert (g.xspec()[1] == 2).all()


def _stereo_x(kind, T, rate, seed):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(T).astype(np.float32) * np.float32(0.2)
    if kind == "same":
        return np.stack([a, a])
    if kind == "inverted":
        return np.stack([a, -a])
    if kind == "half":
        return np.stack([a, a * np.float32(10 ** (-6.02 / 20))])
    if kind == "independent":
        return np.stack([a, rng.standard_normal(T).astype(np.float32) * np.float32(0.2)])
    raise ValueError(kind)


def test_programme_known_answers():
    import meters_lv2_b200 as B
    rate, bins = 48000.0, 2048
    T = int(rate) * 20                                          # the first analyses see the zeroed ring: 20 s keeps that under 0.005 dB
    xs = [_stereo_x(k, T, rate, 750 + i) for i, k in enumerate(("same", "inverted", "half", "independent"))]
    # anti-phase bass under independent highs: a 63 Hz sine in opposite polarity plus independent noise high-passed at 1 kHz
    from scipy.signal import butter, sosfilt
    t = np.arange(T)
    rng = np.random.default_rng(760)
    sos = butter(8, 1000.0, "highpass", fs=rate, output="sos")
    hp = sosfilt(sos, rng.standard_normal((2, T)) * 0.1, axis=1)
    bass = 0.5 * np.sin(2 * np.pi * 63.0 * t / rate)
    xs.append(np.stack([bass + hp[0], -bass + hp[1]]).astype(np.float32))
    # a bin-centred sine of amplitude 0.5 near the 1 kHz band's centre: bin 85 of 4096 points (996.1 Hz)
    f = 85 * rate / (2 * bins)
    sine = (0.5 * np.sin(2 * np.pi * f * t / rate)).astype(np.float32)
    xs.append(np.stack([sine, sine]))
    x = np.concatenate(xs)
    d = B.programme_stereo(x, [T] * len(xs), rate=rate, fft_bins=bins)
    live = np.isfinite(d["band_corr"])
    assert (d["skipped"] == 0).all() and (d["analyses"] == len(X.clock([1024] * (T // 1024) + [T % 1024], bins, rate)[0])).all()
    assert (d["band_corr"][0][live[0]] > 0.9999).all() and (np.abs(d["band_mono_db"][0][live[0]]) < 1e-3).all()
    assert (d["band_corr"][1][live[1]] < -0.9999).all()
    assert (np.abs(d["band_balance_db"][2][live[2]] + 6.02) < 0.01).all()
    above = B.SPEC_BAND_HZ * 2 ** (-1 / 6) >= 250.0
    assert (np.abs(d["band_mono_db"][3][above & live[3]] + 3.0103) < 0.5).all()
    b63 = int(np.argmin(np.abs(B.SPEC_BAND_HZ - 63.0)))
    assert d["band_corr"][4, b63] < -0.99
    hi = B.SPEC_BAND_HZ * 2 ** (-1 / 6) >= 1250.0
    assert (np.abs(d["band_corr"][4][hi & live[4]]) < 0.1).all()
    b1k = int(np.argmin(np.abs(B.SPEC_BAND_HZ - f)))
    assert abs(d["band_level_db"][5, b1k, 0] - 20 * np.log10(0.5)) < 0.01 and abs(d["band_level_db"][5, b1k, 1] + 6.0206) < 0.01
    assert np.array_equal(d["bin_hz"], np.arange(bins) * rate / (2 * bins))


@pytest.mark.parametrize("kind", ["numpy", "cpu_tensor", "cuda_tensor", "callable"])
def test_programme_against_private_banks(kind):
    import torch
    import meters_lv2_b200 as B
    rate, bins, block = 44100.0, 512, 1024
    lens = np.array([0, 1, 5000, 30000, 44100, 12345])
    n = lens.size
    T = int(lens.max())
    x = _signal(n, T, seed=770)
    for i in range(n):
        x[2 * i:2 * i + 2, lens[i]:] = np.nan                   # never read into a result
    src = {"numpy": x, "cpu_tensor": torch.from_numpy(x), "cuda_tensor": torch.from_numpy(x).cuda(),
           "callable": lambda off, nf: x[:, off:off + nf]}[kind]
    grp = [1, 0, 1, -1, 0, 1]
    d = B.programme_stereo(src, lens, rate=rate, fft_bins=bins, block=block, groups=grp)
    for i in range(n):
        p = B.Phasewheel(1, bins, rate); p.xspec_enable()
        if lens[i]:
            _feed(p, np.ascontiguousarray(x[2 * i:2 * i + 2, :lens[i]]), [min(block, lens[i] - o) for o in range(0, lens[i], block)])
        ps, pa, pk = p.xspec()
        p.close()
        assert np.array_equal(U64(ps[0]), U64(d["sums"][i])) and pa[0] == d["analyses"][i] and pk[0] == d["skipped"][i]
    ref = B.stereo_albums(d["sums"], d["analyses"], d["skipped"], grp, rate, bins)
    for f, v in ref.items():
        assert np.array_equal(d[f], v, equal_nan=True), f
    assert list(d["album_n_clips"]) == [2, 3]
    # two shards, gathered in clip order and pooled on the host, pool to the same bits as one bank
    h1 = B.programme_stereo(x[:6], lens[:3], rate=rate, fft_bins=bins, block=block)
    h2 = B.programme_stereo(x[6:], lens[3:], rate=rate, fft_bins=bins, block=block)
    sh = B.stereo_albums(np.concatenate([h1["sums"], h2["sums"]]), np.concatenate([h1["analyses"], h2["analyses"]]),
                         np.concatenate([h1["skipped"], h2["skipped"]]), grp, rate, bins)
    for f, v in sh.items():
        assert np.array_equal(np.asarray(d[f]), np.asarray(v), equal_nan=True), f


def test_argument_errors():
    import meters_lv2_b200 as B
    x = np.zeros((4, 2048), np.float32)
    for kw in (dict(fft_bins=100), dict(fft_bins=16384), dict(block=0), dict(block=8193), dict(rate=10.0)):
        with pytest.raises(B.B200MError):
            B.programme_stereo(x, [2048, 2048], **kw)
    with pytest.raises(B.B200MError):
        B.programme_stereo(x, [], fft_bins=512)
    with pytest.raises(B.B200MError):
        B.programme_stereo(x, [2048, -1], fft_bins=512)
    with pytest.raises(B.B200MError):
        B.programme_stereo(x, [2048, 2048], fft_bins=512, groups=[0])
    L = B.lib()
    assert L.b200m_pw_xspec_enable(None, 1, None) != 0
    g = B.Phasewheel(1, 64)
    g.xspec_enable()
    assert L.b200m_pw_xspec_read(g.h, None, None, None) != 0
