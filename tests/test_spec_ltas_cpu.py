"""CPU: the oracle of the spectrum bank's long-term average spectrum (tests/_spec_ltas.py) on the reference build and on the port,
and the host-side parts of programme_spectrum: the band table, the dB scale and the album pooling helper (spectrum_albums).  No GPU."""
import numpy as np
import pytest

import _oracle as O
import _signals as S
import _spec_ltas as L

HAVE_REF, HAVE_PORT = O.available("reference"), O.available("port")
RATES = [22050.0, 44100.0, 48000.0, 96000.0, 192000.0]
BLOCKS = [1024, 1, 8192, 64, 3, 777, 2048]


def _feed(o, x, blocks, pos=0):
    for n in blocks:
        o.process(x[:, pos:pos + n])
        pos += n
    return pos


@pytest.mark.skipif(not (HAVE_REF and HAVE_PORT), reason="needs oracle/_ref and oracle/liboracle_port.so")
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("nchan", [1, 2])
def test_ltas_on_the_port_equals_the_reference(rate, nchan):
    """the per-frame power summed on copies of the reference build's filter states and on the port's: every block's copies end on
    their oracle's state bit for bit (checked inside process), and the sums and counts agree bit for bit"""
    n = 3
    x = S.nasty(n * nchan, sum(BLOCKS), seed=500 + nchan) * np.float32(0.7)
    x[0, 5000:5100] = 0.0                                    # silence inside a block
    a, b = L.Spectr30(n, nchan, rate, kind="reference"), L.Spectr30(n, nchan, rate, kind="port")
    _feed(a, x, BLOCKS); _feed(b, x, BLOCKS)
    sa, ca = a.ltas(); sb, cb = b.ltas()
    assert np.array_equal(sa.view(np.uint64), sb.view(np.uint64)) and np.array_equal(ca, cb)
    assert np.array_equal(a.read().view(np.uint32), b.read().view(np.uint32))


@pytest.mark.skipif(not (HAVE_REF or HAVE_PORT), reason="needs an oracle build")
def test_ltas_counts_follow_the_finiteness_rule():
    """clean input counts every frame; a NaN or Inf leaves the band's filters non-finite to the end of its block (the scrub runs at
    the end of the run), so those frames are not counted, and the next block counts every frame again"""
    n, nf = 2, 1024
    x = S.white(2 * n, 3 * nf, seed=510)
    x[0, nf + 100] = np.nan                                  # instance 0, block 1, frame 100
    x[3, nf + 1000] = np.inf                                 # instance 1, block 1, frame 1000
    o = L.Spectr30(n, 2)
    _feed(o, x, [nf] * 3)
    _, c = o.ltas()
    assert (c[0] == 2 * nf + 100).all() and (c[1] == 2 * nf + 1000).all(), c[:, :3]
    clean = L.Spectr30(n, 2)
    _feed(clean, S.white(2 * n, 3 * nf, seed=511), [nf] * 3)
    assert (clean.ltas()[1] == 3 * nf).all()


def test_band_centres():
    import meters_lv2_b200 as B
    f = B.SPEC_BAND_HZ
    assert f.shape == (30,) and f[16] == 1000.0
    assert np.allclose(f, [1000.0 * 2.0 ** ((i - 16) / 3.0) for i in range(30)], rtol=0, atol=0)
    assert 24.8 < f[0] < 24.81 and 20.15e3 < f[-1] < 20.16e3


def test_ltas_db_scale_and_floor():
    """10 log10 (2 p) with the level ports' floor: -100 where sqrt (2 p) <= 1e-5, and for NaN (no frame counted)"""
    import meters_lv2_b200 as B
    p = np.array([0.5, 0.005, 5e-11, 4.9e-11, 0.0, np.nan])
    d = B._ltas_db(p)
    assert d[0] == 0.0 and abs(d[1] + 20.0) < 1e-12 and abs(d[2] + 100.0) < 1e-9
    assert list(d[3:]) == [-100.0, -100.0, -100.0]
    s, c = np.array([[3.0, 0.0]]), np.array([[4, 0]])
    lt = B._ltas(s, c)
    assert lt[0, 0] == 0.75 and np.isnan(lt[0, 1])


def _rows(n, seed):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 10 ** 7, size=(n, 30)).astype(np.int64)
    counts[n // 3] = 0                                       # an empty clip
    sums = np.where(counts > 0, rng.random((n, 30)) * counts * 10.0 ** rng.integers(-12, 1, size=(n, 30)), 0.0)
    peak = np.where(counts > 0, rng.uniform(-99, 3, size=(n, 30)), -100.0).astype(np.float32)
    return sums, counts, peak


def test_spectrum_albums_pool_in_clip_order():
    """album sums are the members' sums added one clip at a time in ascending index (bit for bit), counts their sum, the peak the
    largest member's; -1 clips count nowhere, an album without members reads NaN, -100, -100 and 0"""
    import meters_lv2_b200 as B
    n = 41
    sums, counts, peak = _rows(n, 520)
    grp = np.array([(i * 7) % 5 if i % 6 else -1 for i in range(n)], np.int64)
    grp[grp == 3] = 6                                        # albums 3 and 5 empty, 6 the last
    r = B.spectrum_albums(sums, counts, peak, grp)
    g = 7
    assert r["album_ltas"].shape == (g, 30) and r["album_peak_db"].dtype == np.float32
    for a in range(g):
        m = [i for i in range(n) if grp[i] == a]
        assert r["album_n_clips"][a] == len(m)
        if not m:
            assert np.isnan(r["album_ltas"][a]).all() and (r["album_ltas_db"][a] == -100).all() and (r["album_peak_db"][a] == -100).all()
            continue
        for band in (0, 13, 29):
            s = 0.0
            for i in m:
                s += float(sums[i, band])
            c = sum(int(counts[i, band]) for i in m)
            want = s / c if c else np.nan
            got = r["album_ltas"][a, band]
            assert (np.isnan(want) and np.isnan(got)) or np.float64(want).view(np.uint64) == np.float64(got).view(np.uint64), (a, band)
        assert np.array_equal(r["album_peak_db"][a], peak[m].max(axis=0))
    assert np.array_equal(r["album_ltas_db"], B._ltas_db(r["album_ltas"]))


def test_spectrum_albums_of_gathered_shards_equal_one_bank():
    """rows of clips split over two banks (shards), concatenated in clip order as shard.gather_results returns them, pool to the
    same album values bit for bit as the rows of one bank"""
    import meters_lv2_b200 as B
    from meters_lv2_b200 import shard
    n = 50
    sums, counts, peak = _rows(n, 530)
    grp = (np.arange(n) * 11) % 9 - 1
    one = B.spectrum_albums(sums, counts, peak, grp)
    parts = []
    for r in range(2):
        lo, cnt = shard.shard_range(n, r, 2)
        parts += shard.gather_results((sums[lo:lo + cnt], counts[lo:lo + cnt], peak[lo:lo + cnt]))
    two = B.spectrum_albums(*(np.concatenate([p[k] for p in parts]) for k in range(3)), grp)
    for k in one:
        assert np.array_equal(np.asarray(one[k]).view(np.uint8), np.asarray(two[k]).view(np.uint8)), k


def test_spectrum_albums_argument_errors():
    import meters_lv2_b200 as B
    sums, counts, peak = _rows(4, 540)
    with pytest.raises(B.B200MError, match="album ids"):
        B.spectrum_albums(sums, counts, peak, [0, 1, -2, 0])
    with pytest.raises(B.B200MError, match="album ids"):
        B.spectrum_albums(sums, counts, peak, [0, 1])
    with pytest.raises(B.B200MError, match=r"\[N, 30\]"):
        B.spectrum_albums(sums[:, :29], counts, peak, [0, 1, 1, 0])
    r = B.spectrum_albums(sums, counts, peak, [-1, -1, -1, -1])
    assert r["album_ltas"].shape == (0, 30) and r["album_n_clips"].shape == (0,)
