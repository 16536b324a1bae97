"""CPU: the oracle of the needle-meter bank's histogram plane (tests/_ppm_hist.py) on the reference build and on the port, its bin,
limit and run rules at their edges, the library's edge table, and the host-side parts of programme_needle: the derived fields and
the album pooling helper (needle_albums).  No GPU."""
import numpy as np
import pytest

import _oracle as O
import _ppm_hist as H
import _signals as S

HAVE_REF, HAVE_PORT = O.available("reference"), O.available("port")
RATES = [22050, 44100, 48000, 88200, 96000, 176400, 192000]
BLOCKS = [1024, 1, 8192, 64, 3, 777, 2048, 5, 1027]
KINDS = [O.PPM_VU, O.PPM_IEC1, O.PPM_IEC2, O.PPM_MS]


def programme(rows, nfram, seed):
    """rows of white noise whose level swings over 40 dB at different speeds, with a loud burst past 0 dB on the level ports (a
    needle over the default limit) and a quiet row (-90 dBFS) last"""
    x = S.white(rows, nfram, seed=seed)
    t = np.arange(nfram) / max(nfram, 1)
    for r in range(rows):
        x[r] *= np.float32(10.0) ** np.float32(-1.0 + np.sin(np.pi * (r + 1) * t)).astype(np.float32)
    x[0, nfram // 3:nfram // 3 + 9600] *= np.float32(4.0)
    x[rows - 1] *= np.float32(10 ** (-84 / 20))
    return np.ascontiguousarray(x, np.float32)


def _feed(o, x, blocks, pos=0):
    for nf in blocks:
        o.process(x[:, pos:pos + nf])
        pos += nf
    return pos


def _same(a, b):
    (ca, sa), (cb, sb) = a, b
    assert np.array_equal(ca, cb)
    assert np.array_equal(sa.view(np.uint8), sb.view(np.uint8))


@pytest.mark.skipif(not (HAVE_REF and HAVE_PORT), reason="needs oracle/_ref and oracle/liboracle_port.so")
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rate", RATES)
def test_hist_on_the_port_equals_the_reference(rate, kind):
    """the readings counted on copies of the reference build's meters and on the port's: every block's copies end on their oracle's
    state bit for bit (checked inside process), and counts, statistics and readings agree bit for bit"""
    n = 4
    rows = 2 * n if kind == O.PPM_MS else n
    x = programme(rows, sum(BLOCKS), seed=900 + kind)
    a, b = H.Needle(n, kind, rate, oracle="reference"), H.Needle(n, kind, rate, oracle="port")
    _feed(a, x, BLOCKS); _feed(b, x, BLOCKS)
    _same(a.hist(), b.hist())
    assert np.array_equal(a.read().view(np.uint32), b.read().view(np.uint32))
    c, s = a.hist()
    groups = sum(nf // 4 for nf in BLOCKS)
    assert (c.sum(axis=1) == groups).all() and not s["nonfinite"].any()
    if kind in (O.PPM_IEC1, O.PPM_IEC2):                       # the burst drives a peak needle past 0 dB
        assert s["over_groups"][0] > 0 and s["overs"][0] >= 1
    assert (s["peak"] > 0).all() and (s["longest_over"] >= (s["over_groups"] > 0)).all()


@pytest.mark.skipif(not (HAVE_REF or HAVE_PORT), reason="needs an oracle build")
@pytest.mark.parametrize("kind", KINDS)
def test_hist_non_finite_input(kind):
    """NaN, +-Inf, denormals, zeros and clicks: a VU needle goes non-finite on NaN or Inf and an IEC needle on Inf, to the end of the
    block (the clamp at the next call brings it back); those groups count as nonfinite and in no bin, peak stays finite"""
    n, blocks = 3, [1024, 1024, 1, 4096, 333, 1024]
    rows = 2 * n if kind == O.PPM_MS else n
    x = S.nasty(rows, sum(blocks), seed=910 + kind)
    o = H.Needle(n, kind)
    _feed(o, x, blocks)
    c, s = o.hist()
    groups = sum(nf // 4 for nf in blocks)
    assert (c.sum(axis=1) + s["nonfinite"] == groups).all()
    assert s["nonfinite"].sum() > 0 and np.isfinite(s["peak"]).all()
    if HAVE_REF and HAVE_PORT:
        p = H.Needle(n, kind, oracle="port" if o.o.L is O.load("reference") else "reference")
        _feed(p, x, blocks)
        _same(o.hist(), p.hist())


def test_library_edges_equal_numpy():
    """b200m_ppm_hist_edges is float64 10^((-80 + 0.5 k) / 20) rounded to float32, bit for bit; PPM_HIST_EDGES_DB names them"""
    import meters_lv2_b200 as B
    e = B.PPM_HIST_EDGES
    assert e.dtype == np.float32 and e.shape == (241,)
    assert np.array_equal(e.view(np.uint32), H.EDGES.view(np.uint32))
    assert e[0] == np.float32(1e-4) and e[160] == 1.0 and e[200] == 10.0 and e[240] == 100.0 and np.all(np.diff(e) > 0)
    assert np.array_equal(B.PPM_HIST_EDGES_DB, -80.0 + 0.5 * np.arange(241))
    assert B.PPM_HIST_STATS_DTYPE == H.STATS and H.STATS.itemsize == 48


# A meter with w1 = 1, w2 = w3 = 0 (IEC form): each group starts from z1 = z2 = 0 and its first sample a sets z1 = |a| exactly, the
# other three are zero; the group's reading is g * |a|.  So a stream of one nonzero sample per group writes any reading sequence.
def _scripted(a, calls, g=4.0, lim=1.0):
    """run ph_run over readings v = g * a[j] (one group each), split into calls of the given frame counts (their nfram mod 4 tails
    unmetered, filled with full-scale samples that never reach a meter); returns (counts, stats)"""
    a = np.asarray(a, np.float32)
    w = np.array([1.0, 0.0, 0.0, g], np.float32)
    st = np.array([[0, 0, 0, 1]], np.float32)
    c = np.zeros((1, H.BINS), np.uint64); s = H.empty(1)
    k = 0
    for nf in calls:
        x = np.ones((1, nf), np.float32)
        ng = nf // 4
        x[0, :4 * ng] = 0.0
        x[0, 0:4 * ng:4] = a[k:k + ng]
        k += ng
        H.lib().ph_run(1, 1, H._ptr(w), np.float32(lim), 0.0, 0.0, H._ptr(st), H._ptr(x), max(nf, 1), nf, H._ptr(H.EDGES),
                       H._ptr(c), H._ptr(s))
    assert k == len(a)
    return c[0].astype(np.int64), s[0]


def _rules(readings, lim):
    """the plane's statistics, restated over a reading sequence"""
    st = dict(nonfinite=0, over_groups=0, overs=0, longest_over=0, run=0, peak=-np.inf)
    for v in np.asarray(readings, np.float32):
        if not np.isfinite(v):
            st["nonfinite"] += 1
            continue
        st["peak"] = max(st["peak"], v)
        if v >= lim:
            st["over_groups"] += 1
            st["overs"] += st["run"] == 0
            st["run"] += 1
            st["longest_over"] = max(st["longest_over"], st["run"])
        else:
            st["run"] = 0
    return st


def test_readings_at_an_edge_and_at_the_limit():
    """a reading equal to edge k goes to bin k + 1, the float below it to bin k; 0 and the smallest readings go to bin 0, +40 dB and
    above to 241; a reading equal to L is over, the float below it is not"""
    e = H.EDGES
    below = np.nextafter(e, np.float32(0))
    big = np.float32(4e37)
    vals = np.concatenate([e, below, [0.0, np.float32(1e-30), big, np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(0))]])
    vals = vals.astype(np.float32)
    want = np.concatenate([np.arange(1, 242), np.arange(0, 241), [0, 0, 241, 161, 160]])
    for v, k in zip(vals, want):
        c, s = _scripted([v / np.float32(4)], [4])             # g = 4: v / 4 * 4 is v exactly
        assert c.sum() == 1 and c[k] == 1, (v, k, np.argmax(c))
        assert s["over_groups"] == (v >= 1.0) and s["peak"] == v
    c, s = _scripted(np.array([1.0, np.nextafter(np.float32(1.0), np.float32(0))], np.float32) / np.float32(4), [8])
    assert s["over_groups"] == 1 and s["overs"] == 1 and s["run"] == 0 and s["longest_over"] == 1


def test_run_rules_across_calls_tails_and_non_finite_readings():
    """runs continue across calls and unmetered tails; a non-finite reading (g * a overflows) neither starts, extends nor ends a run
    and goes to no bin; the open run counts towards longest_over"""
    big = np.float32(1e38)                                     # g * a = 4e38 overflows to inf
    hi, lo = np.float32(0.5), np.float32(0.125)                # readings 2 and 0.5 against L = 1
    seq = [lo, hi, hi, big, hi, lo, big, lo, hi, big, big, hi, hi, hi, lo, hi, hi, hi, hi, big, hi]
    seq = np.array(seq, np.float32)
    with np.errstate(over="ignore"):
        readings = seq * np.float32(4)
    for calls in ([4 * len(seq)], [4] * len(seq), [6, 9, 4, 17, 7, 4, 13, 4, 12, 5, 12], [84 + 3]):
        assert sum(nf // 4 for nf in calls) == len(seq)
        c, s = _scripted(seq, calls)
        want = _rules(readings, 1.0)
        for k, v in want.items():
            assert s[k] == v, (calls, k, s[k], v)
        assert c.sum() == len(seq) - want["nonfinite"]
    assert want == dict(nonfinite=5, over_groups=12, overs=3, longest_over=5, run=5, peak=np.float32(2.0))


def test_derived_fields():
    import meters_lv2_b200 as B
    h = np.zeros((5, 1, 242), np.int64)
    h[0, 0, 0] = 5; h[0, 0, 161] = 95                          # 95 % reached in bin 161 (0 .. 0.5 dB), 99 % too
    h[1, 0, 0] = 100                                            # everything below -80 dB
    h[2, 0, 100] = 94; h[2, 0, 200] = 5; h[2, 0, 241] = 1       # 95 %: bin 200 (lower edge +19.5 dB), 99 %: bin 200, 100 %: 241
    h[3, 0, 241] = 1
    g, p95, p99 = B._needle_dist(h)
    assert list(g[:, 0]) == [100, 100, 100, 1, 0] and g.dtype == np.int64
    assert p95[0, 0] == 0.0 and p99[0, 0] == 0.0
    assert p95[1, 0] == -np.inf and p99[1, 0] == -np.inf
    assert p95[2, 0] == 19.5 and p99[2, 0] == 19.5
    assert p95[3, 0] == 40.0 and np.isnan(p95[4, 0]) and np.isnan(p99[4, 0])
    assert list(B._peak_db(np.array([1.0, 10.0, 0.0, -1.0, -np.inf], np.float32))) == [0.0, 20.0, -np.inf, -np.inf, -np.inf]


def _rows(n, m, seed):
    rng = np.random.default_rng(seed)
    hist = rng.integers(0, 10 ** 6, size=(n, m, 242)) * (rng.random((n, m, 242)) < 0.2)
    st = np.zeros((n, m), H.STATS)
    for k in ("nonfinite", "over_groups", "overs", "longest_over", "run"):
        st[k] = rng.integers(0, 10 ** 5, size=(n, m))
    st["peak"] = rng.uniform(0, 10, size=(n, m)).astype(np.float32)
    hist[n // 3] = 0; st[n // 3] = H.empty(m)                  # an empty clip
    return hist.astype(np.int64), st


def test_needle_albums_pool_in_clip_order():
    """album counts, nonfinite, over_groups and overs are the members' sums, longest_over and peak their maxima; -1 clips count
    nowhere; an album without members reads 0 counts, -inf peak, NaN percentiles and 0 clips"""
    import meters_lv2_b200 as B
    n, m = 41, 2
    hist, st = _rows(n, m, 920)
    grp = np.array([(i * 7) % 5 if i % 6 else -1 for i in range(n)], np.int64)
    grp[grp == 3] = 6                                          # albums 3 and 5 empty, 6 the last
    r = B.needle_albums(hist, st, grp)
    g = 7
    assert r["album_hist"].shape == (g, m, 242) and r["album_hist"].dtype == np.int64 and r["album_peak"].dtype == np.float32
    for a in range(g):
        mem = [i for i in range(n) if grp[i] == a]
        assert r["album_n_clips"][a] == len(mem)
        if not mem:
            assert not r["album_hist"][a].any() and (r["album_peak"][a] == -np.inf).all() and not r["album_overs"][a].any()
            assert np.isnan(r["album_p95_db"][a]).all() and (r["album_peak_db"][a] == -np.inf).all()
            continue
        assert np.array_equal(r["album_hist"][a], hist[mem].sum(axis=0))
        for k in ("nonfinite", "over_groups", "overs"):
            assert np.array_equal(r["album_" + k][a], st[k][mem].astype(np.int64).sum(axis=0)), k
        assert np.array_equal(r["album_longest_over"][a], st["longest_over"][mem].max(axis=0).astype(np.int64))
        assert np.array_equal(r["album_peak"][a], st["peak"][mem].max(axis=0))
    g2, p95, p99 = B._needle_dist(r["album_hist"])
    assert np.array_equal(r["album_groups"], g2)
    assert np.array_equal(r["album_p95_db"], p95, equal_nan=True) and np.array_equal(r["album_p99_db"], p99, equal_nan=True)


def test_needle_albums_of_gathered_shards_equal_one_bank():
    """rows of clips split over two banks (shards), concatenated in clip order as shard.gather_results returns them, pool to the
    same album values bit for bit as the rows of one bank"""
    import meters_lv2_b200 as B
    from meters_lv2_b200 import shard
    n = 50
    hist, st = _rows(n, 2, 930)
    grp = (np.arange(n) * 11) % 9 - 1
    one = B.needle_albums(hist, st, grp)
    parts = []
    for r in range(2):
        lo, cnt = shard.shard_range(n, r, 2)
        parts += shard.gather_results((hist[lo:lo + cnt], st[lo:lo + cnt]))
    two = B.needle_albums(*(np.concatenate([p[k] for p in parts]) for k in range(2)), grp)
    for k in one:
        assert np.array_equal(np.asarray(one[k]).view(np.uint8), np.asarray(two[k]).view(np.uint8)), k


def test_needle_albums_argument_errors():
    import meters_lv2_b200 as B
    hist, st = _rows(4, 1, 940)
    with pytest.raises(B.B200MError, match="album ids"):
        B.needle_albums(hist, st, [0, 1, -2, 0])
    with pytest.raises(B.B200MError, match="album ids"):
        B.needle_albums(hist, st, [0, 1])
    with pytest.raises(B.B200MError, match=r"\[N, M, 242\]"):
        B.needle_albums(hist[:, :, :241], st, [0, 1, 1, 0])
    with pytest.raises(B.B200MError, match=r"\[N, M, 242\]"):
        B.needle_albums(hist, st["peak"], [0, 1, 1, 0])
    r = B.needle_albums(hist, st, [-1, -1, -1, -1])
    assert r["album_hist"].shape == (0, 1, 242) and r["album_n_clips"].shape == (0,)
