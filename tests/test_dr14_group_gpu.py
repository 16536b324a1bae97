"""GPU: album DR (b200m_dr14_group_reduce / b200m_dr14_group_finish, DR14.group_reduce / group_finish, programme_dr14(groups=)).

An album of tracks that each hold whole 3 s windows and end in a scored one is checked against one reference dr14 instance
(_oracle.Dr14, the reference plugin where oracle/_ref is built) fed the member tracks back to back: m_rms, dr, dr_total and
block_count are bit-identical.  The pooled parts are checked against the members' own state: rows against the numpy sum of their
histograms and window counts, peak2 against the second-largest window peak of their window logs, m_peak against their largest
m_peak port.
"""
import ctypes as C

import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
ALBUM_FIELDS = ("m_rms", "dr", "dr_total", "block_count")


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _win(rate):
    return int(np.rint(np.float32(rate * 3.0))) + 1


def _track(rng, nch, k, w, hazards):
    """k whole windows of noise under a per-window level; hazards: a silent window, NaN and Inf samples inside (never in the last
    window, which stays scored)"""
    lvl = (10.0 ** rng.uniform(-3.0, 0.0, k)).astype(np.float32)
    x = (rng.uniform(-1, 1, (nch, k * w)).astype(np.float32) * np.repeat(lvl, w)[None, :]).astype(np.float32)
    if hazards and k >= 3:
        j = int(rng.integers(0, k - 1))
        x[:, j * w:(j + 1) * w] = 0.0                          # a silent window
        x[0, int(rng.integers(0, (k - 1) * w))] = np.nan
        x[-1, int(rng.integers(0, (k - 1) * w))] = np.inf
    return x


def _library(rng, nch, w, sizes, windows, hazards=True):
    """tracks of the albums sizes[a] (album a), each of windows() whole windows: (x [N * nch, max len], lengths, groups)"""
    tracks, groups = [], []
    for a, s in enumerate(sizes):
        for _ in range(s):
            tracks.append(_track(rng, nch, int(windows()), w, hazards))
            groups.append(a)
    lens = np.array([t.shape[1] for t in tracks], np.int64)
    x = np.zeros((len(tracks) * nch, int(lens.max())), np.float32)
    for i, t in enumerate(tracks):
        x[i * nch:(i + 1) * nch, :t.shape[1]] = t
    return x, lens, np.array(groups, np.int64)


def _back_to_back(x, lens, members, nch, rate):
    """one reference instance fed the member tracks one after another"""
    o = O.Dr14(1, nch, rate, True)
    for i in members:
        t = x[i * nch:(i + 1) * nch, :int(lens[i])]
        for off in range(0, t.shape[1], 8192):
            o.process(np.ascontiguousarray(t[:, off:off + 8192]))
    return o.read()[0]


def _check_vs_reference(alb, a, want, nch, tag):
    got = [alb["m_rms"][a][0], alb["m_rms"][a][1], alb["dr"][a][0], alb["dr"][a][1], alb["dr_total"][a], alb["block_count"][a]]
    cols = [6, 7, 8, 9, 10, 11]
    for g, k in zip(got, cols):
        if k in (7, 9, 10) and nch == 1:
            assert np.isnan(g), (tag, a, k)
            continue
        assert u32(g) == u32(want[k]), (tag, a, k, g, want[k])


def _rows_peaks(bank, G):
    import torch
    rows = torch.empty((G, B().dr14_group_words(bank.nchan)), dtype=torch.int32, device="cuda")
    peaks = torch.empty((G, bank.nchan, 3), dtype=torch.float32, device="cuda")
    return rows, peaks


def B():
    import meters_lv2_b200
    return meters_lv2_b200


@pytest.mark.parametrize("nch", [2, 1])
@pytest.mark.parametrize("rate", [48000.0, 44100.0])
def test_albums_equal_reference_back_to_back(rate, nch):
    """albums of 1..5 tracks of 1..9 windows (albums whose every track has fewer than 3 windows among them), fed as programme_dr14
    ragged blocks; NaN / Inf samples and silent windows inside tracks"""
    w = _win(rate)
    rng = np.random.default_rng(int(rate) + nch)
    sizes = [1, 2, 3, 5, 4, 2, 1]
    x, lens, grp = _library(rng, nch, w, sizes, lambda: rng.integers(1, 10))
    short = grp == 5                                            # album 5: two tracks of 2 windows each, valid only together
    lens_s = np.where(short, 2 * w, lens)
    for i in np.nonzero(short)[0]:
        x[i * nch:(i + 1) * nch, 2 * w:] = 0.0
        x[i * nch:(i + 1) * nch, :2 * w] = _track(rng, nch, 2, w, False)
    lens = lens_s
    res, albums = B().programme_dr14(x, lens, rate, nch, True, block=4096, groups=grp)
    assert (res["dr_total" if nch == 2 else "dr"][short].reshape(2, -1)[:, 0] == 21.0).all()
    alb = albums if nch == 2 else _pad_mono(albums)
    for a in range(len(sizes)):
        want = _back_to_back(x, lens, np.nonzero(grp == a)[0], nch, rate)
        _check_vs_reference(alb, a, want, nch, (rate, nch))
    assert albums["block_count"][5] == 12.0 and albums["dr_total" if nch == 2 else "dr"][5].ravel()[0] < 21.0
    assert np.array_equal(albums["n_tracks"], np.array(sizes))


def _pad_mono(albums):
    nan = np.full((albums["m_rms"].shape[0], 1), np.nan, np.float32)
    return {"m_rms": np.hstack([albums["m_rms"], nan]), "dr": np.hstack([albums["dr"], nan]),
            "dr_total": albums["dr_total"], "block_count": albums["block_count"]}


def _feed(bank, x, lens, block=8192, host=False, stream=None):
    import torch
    for off in range(0, int(lens.max()), block):
        nf = min(block, int(lens.max()) - off)
        xb = np.ascontiguousarray(x[:, off:off + nf])
        lb = np.clip(lens - off, 0, nf)
        if host:
            bank.run(xb, lengths=lb)
        else:
            bank.run(torch.from_numpy(xb).cuda(), lengths=lb, stream=stream)


def _small_bank(rate=48000.0, nch=2, seed=3, log=False):
    w = _win(rate)
    rng = np.random.default_rng(seed)
    x, lens, _ = _library(rng, nch, w, [12], lambda: rng.integers(1, 8))
    lens[3] = 0                                                 # a track that never ran
    bank = B().DR14(len(lens), nch, rate, True)
    if log:
        bank.log_enable(16)
    _feed(bank, x, lens)
    return bank, x, lens


def _np_rows(bank, groups, G):
    nch = bank.nchan
    res = bank.results()
    rows = np.zeros((G, nch * 8000 + 2), np.int64)
    for i, g in enumerate(groups):
        if g >= 0:
            for c in range(nch):
                rows[g, c * 8000:(c + 1) * 8000] += bank.histogram(i, c)
            rows[g, -2] += int(round(float(res["block_count"][i]) / 3.0))
            rows[g, -1] += 1
    return rows


def test_pooled_parts_equal_members():
    """rows = the members' histograms and window counts; peak2 = the second-largest member window peak of the window logs;
    m_peak = the largest member m_peak port; an empty album reads like a fresh plugin; unassigned tracks count nowhere"""
    import torch
    bank, x, lens = _small_bank(log=True)
    pts, cnt, lost = bank.log_drain()
    assert not lost.any()
    res = bank.results()
    groups = np.array([0, 0, 1, 1, 1, -1, 3, 3, 0, -1, 3, 0])   # album 2 empty, album 1 holds the track that never ran
    G = 4
    rows, peaks = _rows_peaks(bank, G)
    bank.group_reduce(groups, rows, peaks)
    alb = bank.group_finish(rows, peaks)
    assert np.array_equal(rows.cpu().numpy().astype(np.int64), _np_rows(bank, groups, G))
    for a in range(G):
        mem = np.nonzero(groups == a)[0]
        for c in range(2):
            wp = [p["peak"][c] for i in mem for p in pts[i][:cnt[i]] if p["silent"] == 0 and not np.isnan(p["peak"][c])]
            nf = sum(int(round(float(res["block_count"][i]) / 3.0)) for i in mem)
            v = sorted(wp + [-80.0, -80.0], reverse=True)
            want = np.float32(v[1]) if nf > 2 else np.float32(-81.0)
            assert u32(alb["peak2"][a][c]) == u32(want), (a, c, alb["peak2"][a][c], want)
            # a track that never ran holds 0 (-80 dB); NaN holds count only if every hold is NaN
            mp = np.where(lens[mem] > 0, res["m_peak"][mem, c], np.float32(-80.0))
            ok = mp[~np.isnan(mp)]
            want_mp = np.float32(-80.0) if mem.size == 0 else (ok.max() if ok.size else np.float32(np.nan))
            assert u32(alb["m_peak"][a][c]) == u32(want_mp), (a, c, alb["m_peak"][a][c], want_mp)
        assert alb["members"][a] == mem.size and alb["windows"][a] == rows[a, -2].item()
    e = alb[2]
    assert (e["m_rms"] == -81).all() and (e["peak2"] == -81).all() and (e["dr"] == 21).all() and e["dr_total"] == 21
    assert e["block_count"] == 0 and (e["m_peak"] == -80).all() and e["windows"] == 0 and e["members"] == 0
    assert not rows[2].any().item() and not peaks[2].any().item()


def test_singleton_albums_equal_tracks_at_full_width():
    """8192 stereo instances of noise at a level drawn per instance and block: G = 8192 singletons reproduce every instance's
    results; the G = 1 row is the sum of the singleton rows"""
    import torch
    bm = B()
    n, nch, rate = 8192, 2, 8000.0
    bank = bm.DR14(n, nch, rate, True)
    gen = torch.Generator(device="cuda"); gen.manual_seed(5)
    for b in range(40):                                          # 40 x 8192 frames: 13 windows of 24001 frames
        lvl = 10.0 ** (torch.rand(n, 1, device="cuda", generator=gen) * -3.0)
        xb = (torch.rand(n * nch, 8192, device="cuda", generator=gen) * 2 - 1) * lvl.repeat_interleave(nch, 0)
        bank.run(xb.contiguous())
    res = bank.results()
    assert (res["block_count"] == 39.0).all()                  # 13 windows each
    rows, peaks = _rows_peaks(bank, n)
    bank.group_reduce(np.arange(n), rows, peaks)
    alb = bank.group_finish(rows, peaks)
    for f in ALBUM_FIELDS + ("m_peak",):
        assert np.array_equal(u32(alb[f]), u32(res[f])), f
    for i in (0, 1, 4097, 8191):
        for c in range(nch):
            assert np.array_equal(rows[i, c * 8000:(c + 1) * 8000].cpu().numpy().astype(np.uint32), bank.histogram(i, c))
    r1, p1 = _rows_peaks(bank, 1)
    bank.group_reduce(np.zeros(n, np.int64), r1, p1)
    assert torch.equal(r1[0].long(), rows.long().sum(0))
    a1 = bank.group_finish(r1, p1)
    assert a1["members"][0] == n and a1["windows"][0] == 13 * n and a1["block_count"][0] == np.float32(3.0 * 13 * n)
    assert np.array_equal(p1[0, :, 0].cpu().numpy(), peaks[:, :, 0].max(0).values.cpu().numpy())
    # a skewed assignment: half the bank in one album, singletons for the rest
    half = n // 2
    gs = np.concatenate([np.zeros(half, np.int64), 1 + np.arange(n - half)])
    rs, ps = _rows_peaks(bank, 1 + n - half)
    bank.group_reduce(gs, rs, ps)
    assert torch.equal(rs[1:], rows[half:]) and torch.equal(rs[0].long(), rows[:half].long().sum(0))


def test_member_list_cache_and_paths():
    """a changing assignment between calls (the member-list cache), host- and device-path banks and a caller stream"""
    import torch
    bm = B()
    rate, nch = 48000.0, 2
    w = _win(rate)
    rng = np.random.default_rng(9)
    x, lens, _ = _library(rng, nch, w, [10], lambda: rng.integers(2, 7))
    hb = bm.DR14(10, nch, rate, True); _feed(hb, x, lens, host=True)
    s = torch.cuda.Stream()
    db = bm.DR14(10, nch, rate, True)
    with torch.cuda.stream(s):
        _feed(db, x, lens, stream=s)
    seq = [(np.array([0, 1, 0, 1, 2, 2, -1, 0, 1, 2]), 3), (np.array([2, 1, 0, 1, 2, 2, -1, 0, 1, 2]), 3),
           (np.array([2, 1, 0, 1, 2, 2, -1, 0, 1, 0]), 3), (np.array([2, 1, 0, 1, 2, 2, -1, 0, 1, 0]), 5),
           (np.array([0, 1, 0, 1, 2, 2, -1, 0, 1, 2]), 3)]
    for groups, G in seq:
        want = _np_rows(hb, groups, G)
        rh, ph = _rows_peaks(hb, G)
        hb.group_reduce(groups, rh, ph)
        ah = hb.group_finish(rh, ph)
        with torch.cuda.stream(s):
            rd, pd = _rows_peaks(db, G)
            db.group_reduce(groups, rd, pd, stream=s)
            ad = db.group_finish(rd, pd, stream=s)
        assert np.array_equal(rh.cpu().numpy().astype(np.int64), want), (groups, G)
        assert np.array_equal(rd.cpu().numpy().astype(np.int64), want), (groups, G)
        assert ah.tobytes() == ad.tobytes()
        assert ph.cpu().numpy().tobytes() == pd.cpu().numpy().tobytes()


def test_unaligned_outputs():
    import torch
    bank, _, _ = _small_bank(seed=4)
    groups = np.array([0, 1, 1, 2, 0, 0, 2, 1, -1, 0, 2, 2])
    G, words = 3, B().dr14_group_words(2)
    rows, peaks = _rows_peaks(bank, G)
    bank.group_reduce(groups, rows, peaks)
    want = bank.group_finish(rows, peaks)
    rb = torch.full((G * words + 2,), -7, dtype=torch.int32, device="cuda")
    pb = torch.full((G * 2 * 3 + 2,), -7.0, dtype=torch.float32, device="cuda")
    r = rb[1:1 + G * words].view(G, words); p = pb[1:1 + G * 6].view(G, 2, 3)
    assert r.data_ptr() % 16 == 4 or r.data_ptr() % 8 == 4
    bank.group_reduce(groups, r, p)
    got = bank.group_finish(r, p)
    assert got.tobytes() == want.tobytes() and torch.equal(r, rows)
    assert p.cpu().numpy().tobytes() == peaks.cpu().numpy().tobytes()
    assert rb[0].item() == -7 and rb[-1].item() == -7 and pb[0].item() == -7.0 and pb[-1].item() == -7.0


def test_shards_equal_one_bank():
    """two banks holding halves of the tracks: rows summed with torch and peaks stacked as two parts equal one bank bit for bit"""
    import torch
    bm = B()
    rate, nch = 44100.0, 2
    w = _win(rate)
    rng = np.random.default_rng(11)
    x, lens, _ = _library(rng, nch, w, [14], lambda: rng.integers(1, 9), hazards=False)   # no NaN hold: an empty part holds 0
    groups = np.array([0, 1, 0, 2, 1, 0, 3, 3, 0, 1, -1, 2, 0, 1])   # album 2 spans both halves, 3 sits in the first only
    G = 5
    one = bm.DR14(14, nch, rate, True); _feed(one, x, lens)
    halves = []
    for lo, hi in ((0, 7), (7, 14)):
        b = bm.DR14(hi - lo, nch, rate, True)
        _feed(b, np.ascontiguousarray(x[lo * nch:hi * nch]), lens[lo:hi])
        r, p = _rows_peaks(b, G)
        b.group_reduce(groups[lo:hi], r, p)
        halves.append((b, r, p))
    r1, p1 = _rows_peaks(one, G)
    one.group_reduce(groups, r1, p1)
    want = one.group_finish(r1, p1)
    rows = halves[0][1] + halves[1][1]
    stack = torch.stack([halves[0][2], halves[1][2]])
    assert torch.equal(rows, r1)
    got = halves[1][0].group_finish(rows, stack)
    assert got.tobytes() == want.tobytes()
    assert one.group_finish(r1, p1.unsqueeze(0)).tobytes() == want.tobytes()


def test_argument_errors_enqueue_nothing():
    import torch
    bm = B()
    bank, _, _ = _small_bank(seed=6)
    tp = bm.DR14(4, 2, 48000.0, False)
    L = bm.lib()
    G = 2
    rows, peaks = _rows_peaks(bank, G)
    g = np.zeros(12, np.uint32)
    rp, pp, st = C.c_void_p(rows.data_ptr()), C.c_void_p(peaks.data_ptr()), bm._stream_ptr(None)
    out = np.empty(G, bm.DR14_ALBUM_DTYPE)
    bad = g.copy(); bad[5] = G
    c0 = bm.launch_count()
    assert L.b200m_dr14_group_reduce(None, bm._np_ptr(g), G, rp, pp, st) == -1
    assert L.b200m_dr14_group_reduce(bank.h, None, G, rp, pp, st) == -1
    assert L.b200m_dr14_group_reduce(bank.h, bm._np_ptr(g), G, None, pp, st) == -1
    assert L.b200m_dr14_group_reduce(bank.h, bm._np_ptr(g), G, rp, None, st) == -1
    assert L.b200m_dr14_group_reduce(bank.h, bm._np_ptr(g), 0, rp, pp, st) == -1
    assert L.b200m_dr14_group_reduce(bank.h, bm._np_ptr(g), bm.DR14_MAX_GROUPS + 1, rp, pp, st) == -1
    assert L.b200m_dr14_group_reduce(bank.h, bm._np_ptr(bad), G, rp, pp, st) == -1
    op = bm._np_ptr(out)
    assert L.b200m_dr14_group_finish(None, rp, pp, 1, G, op, st) == -1
    assert L.b200m_dr14_group_finish(bank.h, None, pp, 1, G, op, st) == -1
    assert L.b200m_dr14_group_finish(bank.h, rp, None, 1, G, op, st) == -1
    assert L.b200m_dr14_group_finish(bank.h, rp, pp, 1, G, None, st) == -1
    assert L.b200m_dr14_group_finish(bank.h, rp, pp, 0, G, op, st) == -1
    assert L.b200m_dr14_group_finish(bank.h, rp, pp, 1, 0, op, st) == -1
    assert L.b200m_dr14_group_finish(bank.h, rp, pp, 1, bm.DR14_MAX_GROUPS + 1, op, st) == -1
    assert bm.launch_count() == c0
    with pytest.raises(bm.B200MError):
        bank.group_reduce(np.zeros(11), rows, peaks)                 # wrong count
    with pytest.raises(bm.B200MError):
        bank.group_reduce(np.zeros(12, np.int64), rows[:, :-1].contiguous(), peaks)
    g4 = np.zeros(4, np.uint32)
    assert L.b200m_dr14_group_reduce(tp.h, bm._np_ptr(g4), G, rp, pp, st) == -4
    assert L.b200m_dr14_group_finish(tp.h, rp, pp, 1, G, op, st) == -4
    assert bm.launch_count() == c0


def test_programme_dr14_albums():
    """programme_dr14(groups=): the album fields equal direct calls on a bank fed alike, dr_mean the numpy mean of the valid track
    dr_total, and every other returned value is the same as without groups"""
    import torch
    bm = B()
    rate, nch = 48000.0, 2
    w = _win(rate)
    rng = np.random.default_rng(17)
    x, lens, _ = _library(rng, nch, w, [20], lambda: rng.integers(1, 8))
    lens[[4, 9]] = [0, w - 5]                                     # a track that never runs, one without a whole window
    groups = rng.integers(-1, 6, 20)
    groups[groups == 4] = 5                                       # album 4 empty
    res, cv, albums = bm.programme_dr14(x, lens, rate, nch, True, block=3000, curves=True, groups=groups)
    res0, cv0 = bm.programme_dr14(x, lens, rate, nch, True, block=3000, curves=True)
    assert res.tobytes() == res0.tobytes()
    for k in cv0:
        assert np.array_equal(cv[k], cv0[k], equal_nan=True), k
    only = bm.programme_dr14(x, lens, rate, nch, True, block=3000)
    assert only.tobytes() == res0.tobytes()
    r2, a2 = bm.programme_dr14(torch.from_numpy(x).cuda(), lens, rate, nch, True, block=3000, groups=groups)
    assert r2.tobytes() == res0.tobytes()
    bank = bm.DR14(20, nch, rate, True)
    _feed(bank, x, lens, block=3000)
    G = int(groups.max()) + 1
    rows, peaks = _rows_peaks(bank, G)
    bank.group_reduce(groups, rows, peaks)
    alb = bank.group_finish(rows, peaks)
    for k in ("m_rms", "peak2", "dr", "m_peak", "dr_total", "block_count"):
        assert np.array_equal(u32(albums[k]), u32(alb[k])), k
        assert np.array_equal(u32(a2[k]), u32(alb[k])), k
    assert np.array_equal(albums["n_windows"], rows[:, -2].cpu().numpy()) and albums["n_windows"].dtype == np.int64
    assert np.array_equal(albums["n_tracks"], np.bincount(groups[groups >= 0], minlength=G))
    for a in range(G):
        v = res0["dr_total"][(groups == a)].astype(np.float64)
        v = v[(v >= 1) & (v <= 20)]
        if v.size:
            assert abs(albums["dr_mean"][a] - v.mean()) <= 1e-12 * abs(v.mean()), a
        else:
            assert np.isnan(albums["dr_mean"][a]), a
    assert np.isnan(albums["dr_mean"][4]) and albums["n_tracks"][4] == 0 and albums["dr_total"][4] == 21.0
    with pytest.raises(bm.B200MError):
        bm.programme_dr14(x, lens, rate, nch, False, groups=groups)
    _, none = bm.programme_dr14(x[:4], lens[:2], rate, nch, True, groups=[-1, -1])
    assert none["dr_total"].shape == (0,) and none["m_rms"].shape == (0, nch)
