"""The true-peak / K-meter histogram plane's rules and its oracle, without a GPU: the reference build against the port at 22.05-192
kHz, non-finite and denormal input, the bin edges, the limit and the square-root threshold rule at their edges, programme_truepeak's
derived fields and the album pooling through needle_albums."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _oracle as O  # noqa: E402
import _tpk_hist as H  # noqa: E402
from _ppm_hist import BINS, EDGES, empty  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import meters_lv2_b200 as B  # noqa: E402

RATES = (22050.0, 44100.0, 48000.0, 88200.0, 96000.0, 176400.0, 192000.0)
need_ref = pytest.mark.skipif(not O.available("reference"), reason="reference oracle not built")


def _sqrt_threshold(e):
    """the least float32 t with sqrtf(t) >= e (the rule the library uses for the K-meter's readings)"""
    e = np.float32(e)
    t = np.float32(np.float64(e) * np.float64(e))
    while np.sqrt(t) < e:
        t = np.nextafter(t, np.float32(np.inf))
    while True:
        d = np.nextafter(t, np.float32(-np.inf))
        with np.errstate(invalid="ignore"):                  # below zero the root is NaN: the loop ends there
            if not np.sqrt(d) >= e:
                return t
        t = d


def _programme(n, nframes, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, nframes)) * rng.uniform(0.05, 1.2, (n, 1))).astype(np.float32)
    x[:, nframes // 3: nframes // 2] *= 3.0                  # a loud passage: overs of -1 dBTP and of the K-meter limit
    return x


def _feed(o, x, block, lengths=None):
    for off in range(0, x.shape[1], block):
        xb = x[:, off:off + block]
        o.process(xb, None if lengths is None else np.clip(np.asarray(lengths) - off, 0, xb.shape[1]))


@need_ref
@pytest.mark.parametrize("fs", RATES)
def test_reference_matches_port(fs):
    x = _programme(3, 3000, int(fs))
    a = H.TpkHist(3, fs, km_limit_db=-30.0, oracle="reference"); b = H.TpkHist(3, fs, km_limit_db=-30.0, oracle="port")
    _feed(a, x, 1000); _feed(b, x, 1000)
    for u, v in zip(a.hist(), b.hist()):
        if u.dtype == np.int64:
            assert np.array_equal(u, v)
        else:
            assert u.tobytes() == v.tobytes()
    tc, ts, kc, ks = a.hist()
    assert ts["over_groups"].sum() > 0 and ks["over_groups"].sum() > 0      # the programme reaches both limits
    assert tc.sum(axis=1).tolist() == [3000 - int(v) for v in ts["nonfinite"]]
    assert kc.sum(axis=1).tolist() == [3 * 250] * 3                          # 1000 // 4 groups per block


def test_nonfinite_and_denormal_input():
    x = _programme(4, 2048, 7) * 0.1
    x[0, 500] = np.nan
    x[1, 900] = np.inf
    x[2, 100:300] = np.float32(1e-41)                        # denormal samples
    x[3, :] = 0.0                                            # digital silence: bin 0
    o = H.TpkHist(4, 48000.0)
    _feed(o, x, 512)
    tc, ts, kc, ks = o.hist()
    assert ts["nonfinite"][0] > 0 and ts["nonfinite"][1] > 0 and ts["nonfinite"][2] == 0 and ts["nonfinite"][3] == 0
    assert ks["nonfinite"][0] > 0 and ks["nonfinite"][2] == 0
    assert tc[3, 0] == 2048 and ts["peak"][3] == 0.0 and kc[3, 0] == 512
    assert (tc.sum(axis=1) + ts["nonfinite"].astype(np.int64) == 2048).all()
    assert (kc.sum(axis=1) + ks["nonfinite"].astype(np.int64) == 512).all()


def test_bin_edges_are_the_needle_planes():
    assert np.array_equal(np.asarray(B.PPM_HIST_EDGES).view(np.uint32), EDGES.view(np.uint32))
    assert B.PPM_HIST_BINS == BINS == EDGES.size + 1


def test_bins_and_limit_at_their_edges():
    """every float within 8 ulps of each edge, and of a limit, lands on the right side"""
    lim = H.limit(-1.0)
    ks = np.arange(-8, 9)
    for e in list(EDGES) + [lim]:
        u = np.array([np.float32(e)], np.float32).view(np.uint32)[0].astype(np.int64) + ks
        u = u.astype(np.uint32).view(np.float32)
        c = np.zeros(BINS, np.uint64); s = empty(1)
        H.count(u, lim, c, s)
        want = np.bincount(np.searchsorted(EDGES, u, side="right"), minlength=BINS)
        assert np.array_equal(c.astype(np.int64), want)
        assert int(s["over_groups"][0]) == int((u >= lim).sum())


def test_sqrt_threshold_rule_at_every_edge():
    """y >= t <=> sqrtf(y) >= e for every float y within 64 ulps of each edge's threshold t (and of a limit's)"""
    ks = np.arange(-64, 65)
    for e in list(EDGES) + [H.limit(-10.0), H.limit(-1.0), np.float32(0.0), np.float32(np.inf)]:
        t = _sqrt_threshold(e)
        if not np.isfinite(t):
            continue
        y = (np.array([t], np.float32).view(np.uint32)[0].astype(np.int64) + ks)
        y = y[y >= 0].astype(np.uint32).view(np.float32)
        assert np.array_equal(np.sqrt(y) >= np.float32(e), y >= t)
    assert _sqrt_threshold(np.float32(np.inf)) == np.inf and _sqrt_threshold(np.float32(0.0)) == 0.0


def test_km_readings_are_binned_in_the_root_domain():
    """a K-meter reading near each edge goes to the bin of its root, as the oracle bins it: sqrtf(2 z2) against e[k]"""
    for k in range(0, 241, 7):
        e = EDGES[k]
        z2 = np.float32(np.float64(e) ** 2 / 2)
        for d in (-2, -1, 0, 1, 2):
            y = np.float32(2.0) * np.array([z2], np.float32).view(np.uint32)[0].astype(np.int64).__add__(d).astype(np.uint32).view(np.float32)
            assert (y >= _sqrt_threshold(e)) == (np.sqrt(y) >= e)


def test_derived_fields():
    rng = np.random.default_rng(3)
    cnt = rng.integers(0, 50, (3, 2, BINS)).astype(np.int64)
    cnt[2, 1] = 0
    st = np.zeros((3, 2), B.PPM_HIST_STATS_DTYPE)
    st["peak"] = -np.inf
    st["peak"][0, 0] = np.float32(0.5)
    st["over_groups"][0, 0] = 480; st["overs"][0, 0] = 3; st["longest_over"][0, 0] = 48; st["nonfinite"][1, 1] = 2
    tp = B._truepeak_fields("tp", cnt, st, 48000.0)
    km = B._truepeak_fields("km", cnt, st, 48000.0)
    assert np.array_equal(tp["tp_frames"], cnt.sum(-1)) and np.array_equal(km["km_groups"], cnt.sum(-1))
    assert tp["tp_over_seconds"][0, 0] == 480 / 48000.0 and km["km_over_seconds"][0, 0] == 4 * 480 / 48000.0
    assert tp["tp_longest_over_s"][0, 0] == 48 / 48000.0 and km["km_longest_over_s"][0, 0] == 4 * 48 / 48000.0
    assert tp["tp_overs"][0, 0] == 3 and tp["tp_nonfinite"][1, 1] == 2
    assert tp["tp_peak_dbtp"][0, 0] == pytest.approx(20 * np.log10(0.5)) and tp["tp_peak_dbtp"][1, 0] == -np.inf
    assert np.isnan(tp["tp_p95_dbtp"][2, 1]) and np.isnan(km["km_p99_db"][2, 1])
    cum = np.cumsum(cnt[0, 0])
    k = int(np.argmax(cum * 100 >= 95 * cnt[0, 0].sum()))
    assert tp["tp_p95_dbtp"][0, 0] == (-np.inf if k == 0 else B.PPM_HIST_EDGES_DB[k - 1])


def test_album_pooling_through_needle_albums():
    x = _programme(6, 2500, 11)
    lengths = np.array([2500, 1200, 0, 2000, 700, 2500])
    o = H.TpkHist(6, 48000.0)
    _feed(o, x, 1024, lengths)
    tc, ts, kc, ks = o.hist()
    grp = np.array([0, 0, 1, -1, 1, 0])
    out = B._truepeak_fields("tp", tc.reshape(6, 1, BINS), ts.reshape(6, 1), 48000.0, grp)
    a = out["tp_album_hist"]
    assert np.array_equal(a[0, 0], tc[[0, 1, 5]].sum(0)) and np.array_equal(a[1, 0], tc[[2, 4]].sum(0))
    assert out["tp_album_overs"][0, 0] == int(ts["overs"][[0, 1, 5]].sum())
    assert out["tp_album_peak"][0, 0] == ts["peak"][[0, 1, 5]].max()
    assert out["tp_album_n_clips"].tolist() == [3, 2]
    # two shards pool to the same result as one bank
    s1 = B._truepeak_fields("km", kc[:3].reshape(3, 1, BINS), ks[:3].reshape(3, 1), 48000.0)
    s2 = B._truepeak_fields("km", kc[3:].reshape(3, 1, BINS), ks[3:].reshape(3, 1), 48000.0)
    pooled = B.needle_albums(np.concatenate([s1["km_hist"], s2["km_hist"]]), np.concatenate([s1["km_stats"], s2["km_stats"]]), grp)
    one = B.needle_albums(kc.reshape(6, 1, BINS), ks.reshape(6, 1), grp)
    for k in one:
        assert np.array_equal(one[k], pooled[k], equal_nan=True)
    assert o.hist()[1]["nonfinite"][2] == 0 and o.hist()[0][2].sum() == 0    # a clip of length 0 adds nothing
