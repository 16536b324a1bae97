"""CPU: the oracle of the correlation bank's histogram plane (tests/_cor_hist.py) on the reference build and on the port, its bin
and gate rules at their edges, and the host-side parts of programme_correlation: the derived fields and the album pooling helper
(correlation_albums).  No GPU."""
import ctypes as C

import numpy as np
import pytest

import _cor_hist as H
import _oracle as O
import _signals as S

HAVE_REF, HAVE_PORT = O.available("reference"), O.available("port")
RATES = [22050, 44100, 48000, 88200, 96000, 176400, 192000]
BLOCKS = [1024, 1, 8192, 64, 3, 777, 2048]


def stereo(n, nfram, seed):
    """n pairs whose correlation sweeps from +1 to -1 and back at different speeds: R = c L + s N with c = cos (phase), a quiet pair
    (-90 dBFS, under the default gate) last"""
    a, b = S.white(n, nfram, seed=seed), S.white(n, nfram, seed=seed + 1)
    t = np.arange(nfram) / nfram
    x = np.empty((2 * n, nfram), np.float32)
    for i in range(n):
        ph = np.pi * (i + 1) * t
        x[2 * i] = a[i]
        x[2 * i + 1] = (np.cos(ph) * a[i] + np.sin(ph) * b[i]).astype(np.float32)
    x[2 * n - 2:] *= np.float32(10 ** (-84 / 20))
    return x


def _feed(o, x, blocks, pos=0):
    for nf in blocks:
        o.process(x[:, pos:pos + nf])
        pos += nf
    return pos


@pytest.mark.skipif(not (HAVE_REF and HAVE_PORT), reason="needs oracle/_ref and oracle/liboracle_port.so")
@pytest.mark.parametrize("tcf", [0.3, 1.0])
@pytest.mark.parametrize("rate", RATES)
def test_hist_on_the_port_equals_the_reference(rate, tcf):
    """the readings counted on copies of the reference build's states and on the port's: every block's copies end on their
    oracle's state bit for bit (checked inside process), and counts and sums agree bit for bit"""
    n = 4
    x = stereo(n, sum(BLOCKS), seed=700)
    x[2, 5000:5100] = 0.0                                    # silence inside a block
    a, b = H.Stcorr(n, rate, tcf=tcf, kind="reference"), H.Stcorr(n, rate, tcf=tcf, kind="port")
    _feed(a, x, BLOCKS); _feed(b, x, BLOCKS)
    ca, sa = a.hist(); cb, sb = b.hist()
    assert np.array_equal(ca, cb) and np.array_equal(sa.view(np.uint64), sb.view(np.uint64))
    assert np.array_equal(a.read().view(np.uint32), b.read().view(np.uint32))
    assert (ca[:n - 1].sum(axis=1) > 0.9 * sum(BLOCKS)).all() and ca[n - 1].sum() == 0    # the quiet pair stays under the gate
    assert (ca[:n - 1, :100].sum(axis=1) > 0).all() and (ca[:n - 1, 100:].sum(axis=1) > 0).all()


@pytest.mark.skipif(not (HAVE_REF or HAVE_PORT), reason="needs an oracle build")
def test_hist_non_finite_input():
    """a NaN or Inf leaves the pair's state non-finite to the end of its block (the scrub runs at block end), so its readings are not
    counted there, and the next block counts every frame again; denormals and zeros count like any sample (no gate)"""
    n, nf = 3, 1024
    x = stereo(n, 3 * nf, seed=710)
    x[0, nf + 100] = np.nan                                  # pair 0, block 1, frame 100
    x[3, nf + 1000] = np.inf                                 # pair 1, block 1, frame 1000
    x[4, 10:20] = np.float32(1e-42); x[5, 30:40] = 0.0       # pair 2: denormals and zeros
    o = H.Stcorr(n, gate_db=-np.inf)
    _feed(o, x, [nf] * 3)
    c, s = o.hist()
    assert list(c.sum(axis=1)) == [2 * nf + 100, 2 * nf + 1000, 3 * nf] and np.isfinite(s).all()
    if HAVE_REF and HAVE_PORT:
        p = H.Stcorr(n, gate_db=-np.inf, kind="port" if o.o.L is O.load("reference") else "reference")
        _feed(p, x, [nf] * 3)
        cp, sp = p.hist()
        assert np.array_equal(c, cp) and np.array_equal(s.view(np.uint64), sp.view(np.uint64))


def _one_frame(states, thr):
    """ch_run over one frame with w1 = w2 = 0: the states stay put (|zl|, |zr| >= 1 absorb the 1e-20), so the frame's reading and
    gate are those of the given zlr, zll, zrr"""
    st = np.ascontiguousarray(states, np.float32)
    n = st.shape[0]
    x = np.zeros((2 * n, 1), np.float32)
    c = np.zeros((n, H.BINS), np.uint64); s = np.zeros(n, np.float64)
    H.lib().ch_run(n, 0.0, 0.0, C.c_float(thr), H._ptr(st), H._ptr(x), 1, 1, H._ptr(c), H._ptr(s))
    return c.astype(np.int64), s


def _bin(r):
    with np.errstate(over="ignore"):
        k = np.floor(np.float32(np.float32(r) + np.float32(1.0)) * np.float32(100.0))
    return int(min(max(k, 0.0), 199.0))


def test_bin_rule_at_its_edges():
    """with zll = zrr = 1 the reading is zlr exactly: -1 -> bin 0, 0 -> 100, 1 -> 199 (clamped), past +-1 clamped, readings just
    below 0 fall in 99 or, where r + 1 rounds to 1, in 100; the rule is the fp32 statement of the bank's header"""
    tiny = np.nextafter(np.float32(0), np.float32(-1))
    rs = np.array([-1.0, 0.0, 1.0, -0.004, -6e-8, -2e-8, tiny, 1.5, -3.0, 0.99, -0.99, 0.005, 3.4e38, -3.4e38], np.float32)
    edges = np.float32(np.arange(-100, 100) / 100.0)
    rs = np.concatenate([rs, edges])
    st = np.zeros((rs.size, 5), np.float32)
    st[:, 0] = st[:, 1] = 1.0; st[:, 2] = rs; st[:, 3] = st[:, 4] = 1.0
    c, s = _one_frame(st, 0.0)
    got = np.argmax(c, axis=1)
    assert (c.sum(axis=1) == 1).all()
    assert list(got[:10]) == [0, 100, 199, 99, 99, 100, 100, 199, 0, 199]     # fp32 0.99 is 0.99000001
    assert list(got[10:14]) == [0, 100, 199, 0]
    assert list(got) == [_bin(r) for r in rs]
    assert np.array_equal(s, rs.astype(np.float64))
    import meters_lv2_b200 as B
    e = B.COR_HIST_EDGES
    assert e.shape == (201,) and e[0] == -1.0 and e[100] == 0.0 and e[200] == 1.0 and np.all(np.diff(e) > 0)
    # the float32 nearest each lower edge falls in that bin or, where it lies below the edge, in the one before
    assert (np.abs(got[14:] - np.arange(200)) <= 1).all()


def test_gate_at_thr_at_minus_inf_and_on_silence():
    thr = H.gate(-70.0)
    assert thr == np.float32(2e-7) and H.gate(-np.inf) == 0.0
    below = np.nextafter(thr, np.float32(0))
    st = np.array([[1, 1, 0, thr, 0], [1, 1, 0, below, 0], [1, 1, 0, thr / 2, thr / 2], [1, 1, 0, 0, 0]], np.float32)
    c, _ = _one_frame(st, thr)
    assert list(c.sum(axis=1)) == [1, 0, 1, 0]
    c, _ = _one_frame(st, 0.0)
    assert list(c.sum(axis=1)) == [1, 1, 1, 1] and (c[:, 100] == 1).all()
    nan = np.array([[1, 1, np.nan, 1, 1], [1, 1, 1, np.inf, 1]], np.float32)
    c, s = _one_frame(nan, 0.0)
    assert not c.any() and not s.any()                       # a non-finite reading never counts, whatever the gate
    # digital silence: the bias floor (about -88 dB at 1024-frame blocks) stays under the default gate; without a gate every
    # frame counts, near r = 0
    x = np.zeros((2, 40 * 1024), np.float32)
    for g, want in ((-70.0, 0), (-np.inf, x.shape[1])):
        o = H.Stcorr(1, gate_db=g)
        _feed(o, x, [1024] * 40)
        c, _ = o.hist()
        assert c.sum() == want, g
    assert (c[0, 99:101].sum() == c.sum())


def test_derived_fields():
    import meters_lv2_b200 as B
    h = np.zeros((4, 200), np.int64)
    h[0, 0] = 1; h[0, 150] = 99                              # 1 % reached in bin 0, 5 % in bin 150
    h[1, 199] = 7
    h[2, 99] = 3; h[2, 100] = 1
    s = np.array([-1.0 + 99 * 0.505, 7.0, -0.01, 0.0])
    d = B._cor_dist(h, s)
    assert list(d["frames"]) == [100, 7, 4, 0] and d["frames"].dtype == np.int64
    assert d["p1"][0] == -1.0 and d["p5"][0] == 0.5 and d["p1"][1] == 0.99 and d["p1"][2] == -0.01 and d["p5"][2] == -0.01
    assert d["below0"][0] == 0.01 and d["below0"][1] == 0.0 and d["below0"][2] == 0.75
    assert d["mean"][1] == 1.0 and d["mean"][2] == -0.0025
    assert all(np.isnan(d[k][3]) for k in ("mean", "below0", "p1", "p5"))


def _rows(n, seed):
    rng = np.random.default_rng(seed)
    hist = rng.integers(0, 10 ** 6, size=(n, 200)) * (rng.random((n, 200)) < 0.3)
    hist[n // 3] = 0                                         # an empty clip
    fr = hist.sum(axis=1)
    sums = np.where(fr > 0, rng.uniform(-1, 1, size=n) * fr, 0.0) * (1 + rng.random(n) * 1e-9)
    return hist.astype(np.int64), sums


def test_correlation_albums_pool_in_clip_order():
    """album sums are the members' sums added one clip at a time in ascending index (bit for bit), counts their sum; -1 clips count
    nowhere, an album without members reads 0 frames, NaN fields and 0 clips"""
    import meters_lv2_b200 as B
    n = 41
    hist, sums = _rows(n, 720)
    grp = np.array([(i * 7) % 5 if i % 6 else -1 for i in range(n)], np.int64)
    grp[grp == 3] = 6                                        # albums 3 and 5 empty, 6 the last
    r = B.correlation_albums(hist, sums, grp)
    g = 7
    assert r["album_hist"].shape == (g, 200) and r["album_hist"].dtype == np.int64 and r["album_sums"].shape == (g,)
    for a in range(g):
        m = [i for i in range(n) if grp[i] == a]
        assert r["album_n_clips"][a] == len(m)
        if not m:
            assert r["album_frames"][a] == 0 and not r["album_hist"][a].any() and r["album_sums"][a] == 0
            assert all(np.isnan(r[k][a]) for k in ("album_mean", "album_below0", "album_p1", "album_p5"))
            continue
        s = 0.0
        for i in m:
            s += float(sums[i])
        assert np.float64(s).view(np.uint64) == r["album_sums"][a].view(np.uint64), a
        assert np.array_equal(r["album_hist"][a], hist[m].sum(axis=0))
    d = B._cor_dist(r["album_hist"], r["album_sums"])
    for k in ("frames", "mean", "below0", "p1", "p5"):
        assert np.array_equal(r["album_" + k], d[k], equal_nan=True), k


def test_correlation_albums_of_gathered_shards_equal_one_bank():
    """rows of clips split over two banks (shards), concatenated in clip order as shard.gather_results returns them, pool to the
    same album values bit for bit as the rows of one bank"""
    import meters_lv2_b200 as B
    from meters_lv2_b200 import shard
    n = 50
    hist, sums = _rows(n, 730)
    grp = (np.arange(n) * 11) % 9 - 1
    one = B.correlation_albums(hist, sums, grp)
    parts = []
    for r in range(2):
        lo, cnt = shard.shard_range(n, r, 2)
        parts += shard.gather_results((hist[lo:lo + cnt], sums[lo:lo + cnt]))
    two = B.correlation_albums(*(np.concatenate([p[k] for p in parts]) for k in range(2)), grp)
    for k in one:
        assert np.array_equal(np.asarray(one[k]).view(np.uint8), np.asarray(two[k]).view(np.uint8)), k


def test_correlation_albums_argument_errors():
    import meters_lv2_b200 as B
    hist, sums = _rows(4, 740)
    with pytest.raises(B.B200MError, match="album ids"):
        B.correlation_albums(hist, sums, [0, 1, -2, 0])
    with pytest.raises(B.B200MError, match="album ids"):
        B.correlation_albums(hist, sums, [0, 1])
    with pytest.raises(B.B200MError, match=r"\[N, 200\]"):
        B.correlation_albums(hist[:, :199], sums, [0, 1, 1, 0])
    r = B.correlation_albums(hist, sums, [-1, -1, -1, -1])
    assert r["album_hist"].shape == (0, 200) and r["album_n_clips"].shape == (0,)
