"""GPU: the needle-meter bank's histogram plane (b200m_ppm_hist_*, NeedleMeters.hist_enable / hist) and programme_needle, against
the oracle of tests/_ppm_hist.py (the per-group readings of the reference build's own needles, with the plane's bin, limit and run
rules)."""
import ctypes as C

import numpy as np
import pytest

import _oracle as O
import _ppm_hist as H
import _signals as S
from test_ppm_hist_cpu import programme

pytestmark = pytest.mark.gpu
KINDS = [O.PPM_VU, O.PPM_IEC1, O.PPM_IEC2, O.PPM_MS]


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_hist(tag, got, want):
    (gc, gs), (wc, ws) = got, want
    assert np.array_equal(gc, wc), (tag, np.argwhere(gc != wc)[:4])
    assert np.array_equal(gs.view(np.uint8), ws.view(np.uint8)), (tag, gs, ws)


def _same_bank(tag, a, b, stream=None):
    """ports and the four states of two banks bit for bit"""
    assert np.array_equal(u32(a.state(stream)), u32(b.state(stream))), tag
    assert np.array_equal(u32(a.read(stream)), u32(b.read(stream))), tag


def _rows(kind, n):
    return 2 * n if kind == O.PPM_MS else n


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rate,n,blocks", [
    (48000, 37, [1024] * 4 + [1, 2, 3, 5, 1027, 8192, 64]),
    (22050, 6, [1024, 8192, 1, 333, 2, 1027]),
    (44100, 9, [1024] * 3 + [8192, 5, 441, 3]),
    (96000, 3, [8192, 1, 4096, 7, 1027]),
    (192000, 2, [8192, 8192, 1, 1920, 5]),
])
def test_hist_bit_exact_with_ports_unchanged(kind, rate, n, blocks):
    """counts and statistics bit-identical to the oracle after every block; ports and states bit-identical with the plane on, off and
    in the reference build"""
    import torch
    import meters_lv2_b200 as B
    x = programme(_rows(kind, n), sum(blocks), seed=1000 + n + kind)
    on, off = B.NeedleMeters(n, kind, rate), B.NeedleMeters(n, kind, rate)
    on.hist_enable()
    o = H.Needle(n, kind, rate)
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for b, nf in enumerate(blocks):
        on.process(xd[:, pos:pos + nf]); off.process(xd[:, pos:pos + nf]); o.process(x[:, pos:pos + nf])
        pos += nf
        _same_hist(b, on.hist(), o.hist())
        assert np.array_equal(u32(on.state()), u32(o.peek())), b
        assert np.array_equal(u32(off.state()), u32(o.peek())), b
        if b % 3 == 2:                                         # read() now and then: _res resets the port's maximum, not the plane
            p = o.read()
            assert np.array_equal(u32(on.read()), u32(p)) and np.array_equal(u32(off.read()), u32(p)), b
    _same_bank("end", on, off)
    c, s = on.hist()
    assert (c.sum(axis=1) == sum(nf // 4 for nf in blocks)).all() and not s["nonfinite"].any()


@pytest.mark.parametrize("kind", KINDS)
def test_hist_non_finite_input(kind):
    """NaN, +-Inf, denormals, zeros and clicks (host path): nonfinite counts the groups whose reading is not finite, as in the oracle,
    peak ignores them, and the ports still equal the reference's"""
    import meters_lv2_b200 as B
    n, blocks = 5, [1024, 1024, 1, 4096, 333, 1024]
    x = S.nasty(_rows(kind, n), sum(blocks), seed=1020 + kind)
    g = B.NeedleMeters(n, kind); g.hist_enable(limit_db=-20.0)
    o = H.Needle(n, kind, limit_db=-20.0)
    pos = 0
    for nf in blocks:
        blk = np.ascontiguousarray(x[:, pos:pos + nf])
        g.process(blk); o.process(blk)
        pos += nf
        _same_hist(pos, g.hist(), o.hist())
        assert np.array_equal(u32(g.read()), u32(o.read()))
    c, s = g.hist()
    assert s["nonfinite"].sum() > 0 and np.isfinite(s["peak"]).all()
    assert (c.sum(axis=1) + s["nonfinite"] == sum(nf // 4 for nf in blocks)).all()


@pytest.mark.parametrize("kind", [O.PPM_IEC2, O.PPM_MS, O.PPM_VU])
def test_hist_ragged_paths_clear_and_enable(kind):
    """ragged blocks (lengths 0 included) against private oracle meters fed only their own frames, with an over run that spans a
    zero-length hold; the host path, the device path on a caller stream and switches between them; clear(unit) zeroes that unit's
    rows only (both of an M/S pair), clear() every row; disabling freezes the counts and keeps the ports going, enabling again zeroes
    every row and sets the new limit"""
    import torch
    import meters_lv2_b200 as B
    n = 11
    per = 2 if kind == O.PPM_MS else 1
    rng = np.random.default_rng(1030 + kind)
    sizes = [1024, 512, 8192, 1, 1024, 700, 1024, 2048, 64, 1024, 1024, 300, 4096]
    x = programme(_rows(kind, n), sum(sizes), seed=1031)
    x[:per] = S.sine(sum(sizes), 1000.0, amp=0.9)              # unit 0: a steady tone, over -20 dB all along
    g = B.NeedleMeters(n, kind)
    st = torch.cuda.Stream()
    g.hist_enable(limit_db=-20.0, stream=st)
    priv = [H.Needle(1, kind, limit_db=-20.0) for _ in range(n)]
    counting = True

    def want():
        return np.concatenate([p.hist()[0] for p in priv]), np.concatenate([p.hist()[1] for p in priv])

    pos = 0
    for b, nf in enumerate(sizes):
        ln = rng.integers(0, nf + 1, size=n)
        ln[b % n] = 0
        ln[(b + 3) % n] = nf
        ln[0] = 0 if b == 5 else nf                             # unit 0's over run spans a hold
        blk = x[:, pos:pos + nf]
        host = b % 3 == 1
        if host:
            g.process(np.ascontiguousarray(blk), lengths=ln)
        else:
            with torch.cuda.stream(st):
                xd = torch.from_numpy(np.ascontiguousarray(blk)).cuda()
            g.process(xd, stream=st, lengths=ln)
        before = [p.hist() for p in priv]
        for i in range(n):
            if ln[i]:
                priv[i].process(blk[per * i:per * i + per, :ln[i]])
        if not counting:                                       # the plane is off: the private oracles' counts stay put
            for p, (c0, s0) in zip(priv, before):
                p.counts[:] = c0; p.stats = s0
        pos += nf
        rs = None if host else st
        if counting:
            _same_hist(b, g.hist(stream=rs), want())
        assert np.array_equal(u32(g.state(stream=rs)), u32(np.concatenate([p.peek() for p in priv]))), b
        if b == 4:
            before = g.hist(stream=rs)
            g.clear(3, stream=rs)
            priv[3] = H.Needle(1, kind, limit_db=-20.0)
            after = g.hist(stream=rs)
            rows = np.arange(per * 3, per * 4)
            assert not after[0][rows].any() and (after[1]["peak"][rows] == -np.inf).all() and not after[1]["over_groups"][rows].any()
            keep = np.ones(n * per, bool); keep[rows] = False
            assert np.array_equal(after[0][keep], before[0][keep]) and np.array_equal(after[1][keep], before[1][keep])
        if b == 6:                                             # one run since the needle first passed the limit, across the hold
            s0 = g.hist(stream=rs)[1]
            assert s0["overs"][0] == 1 and s0["run"][0] == s0["over_groups"][0] == s0["longest_over"][0] > 0
            g.clear(stream=rs)
            priv = [H.Needle(1, kind, limit_db=-20.0) for _ in range(n)]
            c, s = g.hist(stream=rs)
            assert not c.any() and (s["peak"] == -np.inf).all() and not s["run"].any()
        if b == 7:
            g.hist_enable(False, stream=rs)
            counting = False
            with pytest.raises(B.B200MError, match="histogram plane is off"):
                g.hist(stream=rs)
        if b == 9:
            g.hist_enable(limit_db=-6.0, stream=rs)
            counting = True
            for p in priv:
                p.clear_hist(-6.0)
            c, s = g.hist(stream=rs)
            assert not c.any() and (s["peak"] == -np.inf).all()


def test_known_answers():
    """three 0.5 s tone bursts 6 dB above the limit, 2 s apart, give three overs on an IEC II meter (its needle falls 6 dB in about
    0.7 s); each over lasts the burst plus the fall to the limit (the rise takes milliseconds); a steady tone's peak equals read()"""
    import torch
    import meters_lv2_b200 as B
    fs, block = 48000, 1024
    tone = S.sine(fs, 1000.0, amp=0.5)
    ref = B.NeedleMeters(1, O.PPM_IEC2)
    for k in range(fs // block):
        ref.process(np.ascontiguousarray(tone[None, k * block:(k + 1) * block]))
    steady_db = 20 * np.log10(float(ref.read()[0]))
    nf = 7 * fs
    x = np.zeros((1, nf), np.float32)
    for k in range(3):
        a = fs // 2 + 2 * k * fs
        x[0, a:a + fs // 2] = S.sine(fs // 2, 1000.0, amp=0.5)
    g = B.NeedleMeters(1, O.PPM_IEC2)
    g.hist_enable(limit_db=steady_db - 6.0)
    xd = torch.from_numpy(x).cuda()
    for off in range(0, nf, block):
        g.process(xd[:, off:off + block])
    c, s = g.hist()
    assert s["overs"][0] == 3 and s["run"][0] == 0
    over_s = 4.0 * s["over_groups"][0] / fs
    assert 3 * 0.5 - 0.03 <= over_s <= 3 * (0.5 + 0.8), over_s
    assert 0.5 - 0.01 <= 4.0 * s["longest_over"][0] / fs <= 0.5 + 0.8
    # steady tone: the reading read() returns is the largest group reading
    t = B.NeedleMeters(4, O.PPM_VU)
    t.hist_enable()
    xt = np.stack([S.sine(3 * fs, f, amp=a) for f, a in ((1000.0, 0.5), (440.0, 0.1), (5000.0, 0.9), (60.0, 0.01))])
    for off in range(0, xt.shape[1], block):
        t.process(np.ascontiguousarray(xt[:, off:off + block]))
    _, st = t.hist()
    assert np.array_equal(u32(st["peak"]), u32(t.read()))


def _clips(rows_per, lengths, seed, kind):
    n = len(lengths)
    x = programme(rows_per * n, int(max(lengths)) + 5, seed=seed)
    for i in range(n):
        x[rows_per * i:rows_per * (i + 1), lengths[i]:] = np.nan   # past a clip's end: never read into a result
    return x


def _private(x, lengths, kind, per, block, limit_db, gains=(-6.0, -6.0)):
    """each clip fed alone to a NeedleMeters with the plane on in `block`-frame pieces"""
    import meters_lv2_b200 as B
    c, s, rd = [], [], []
    for i, ln in enumerate(lengths):
        m = B.NeedleMeters(1 if kind == O.PPM_MS else per, kind)
        if kind == O.PPM_MS:
            m.set_gain(*gains)
        m.hist_enable(limit_db=limit_db)
        for off in range(0, int(ln), block):
            m.process(np.ascontiguousarray(x[per * i:per * i + per, off:min(off + block, ln)]))
        a, b = m.hist()
        c.append(a); s.append(b); rd.append(m.read())
        m.close()
    return np.array(c), np.array(s), np.array(rd, np.float32)


@pytest.mark.parametrize("kind,nchan,block,limit_db", [
    (O.PPM_VU, 2, 1024, -10.0), (O.PPM_IEC1, 1, 777, -10.0), (O.PPM_IEC2, 2, 1024, -3.0), (O.PPM_MS, 2, 1027, -12.0),
    (O.PPM_IEC2, 3, 4096, np.inf),
])
def test_programme_needle_equals_private_meters(kind, nchan, block, limit_db):
    import meters_lv2_b200 as B
    lengths = np.array([40000, 0, 1024, 1, 90000, 777, 2 * 777, 12345, 50, 6])
    per = 2 if kind == O.PPM_MS else nchan
    x = _clips(per, lengths, 1040 + kind, kind)
    r = B.programme_needle(x, lengths, kind, nchan=nchan, limit_db=limit_db, block=block)
    c, s, rd = _private(x, lengths, kind, per, block, limit_db)
    assert np.array_equal(r["hist"], c) and np.array_equal(r["stats"].view(np.uint8), s.view(np.uint8))
    assert np.array_equal(u32(r["reading"]), u32(rd))
    assert r["hist"].shape == (lengths.size, per, 242) and r["reading"].dtype == np.float32
    g, p95, p99 = B._needle_dist(c)
    assert np.array_equal(r["groups"], g) and np.array_equal(r["p95_db"], p95, equal_nan=True)
    assert np.array_equal(r["p99_db"], p99, equal_nan=True)
    assert np.array_equal(r["groups"][:, 0], [ln // block * (block // 4) + (ln % block) // 4 for ln in lengths])
    assert np.array_equal(r["seconds"], r["groups"].astype(np.float64) * 4.0 / 48000.0)
    assert np.array_equal(r["over_seconds"], s["over_groups"].astype(np.float64) * 4.0 / 48000.0)
    assert np.array_equal(r["longest_over_s"], s["longest_over"].astype(np.float64) * 4.0 / 48000.0)
    assert np.array_equal(r["overs"], s["overs"]) and np.array_equal(r["nonfinite"], s["nonfinite"])
    assert np.array_equal(u32(r["peak"]), u32(s["peak"])) and np.array_equal(r["peak_db"], B._peak_db(s["peak"]))
    assert r["groups"][1].sum() == 0 and r["reading"][1].sum() == 0 and (r["peak"][1] == -np.inf).all()
    assert np.isnan(r["p95_db"][1]).all()
    if limit_db == np.inf:
        assert not r["over_groups"].any()
    elif kind != O.PPM_MS:
        assert r["overs"].sum() > 0


def test_programme_needle_inputs_albums_and_shards():
    """numpy, CUDA-tensor and callable inputs give the same bits; albums with unassigned clips and empty albums are needle_albums of
    the clip rows; two banks' rows pooled give the one bank's album values bit for bit; M/S gains reach the meters"""
    import torch
    import meters_lv2_b200 as B
    lengths = np.array([3000, 50000, 0, 1024, 4097, 10, 20480, 6000, 333, 4500, 1])
    n = lengths.size
    x = _clips(2, lengths, 1050, O.PPM_MS)
    grp = np.array([0, 2, 0, -1, 2, 4, 0, -1, 2, 4, 0])        # albums 1 and 3 have no members
    for kind in (O.PPM_IEC1, O.PPM_MS):
        ref = B.programme_needle(x, lengths, kind, limit_db=-12.0, groups=grp)
        xd = torch.from_numpy(x).cuda()
        for tag, inp in (("cpu tensor", torch.from_numpy(x)), ("cuda", xd), ("callable", lambda off, nf: xd[:, off:off + nf])):
            r = B.programme_needle(inp, lengths, kind, limit_db=-12.0, groups=grp)
            assert set(r) == set(ref), tag
            for k in ref:
                assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(ref[k]).view(np.uint8)), (tag, k)
        alb = B.needle_albums(ref["hist"], ref["stats"], grp)
        for k in alb:
            assert np.array_equal(np.asarray(ref[k]).view(np.uint8), np.asarray(alb[k]).view(np.uint8)), k
        assert list(ref["album_n_clips"]) == [4, 0, 3, 0, 2]
        assert not ref["album_groups"][[1, 3]].any() and (ref["album_peak"][[1, 3]] == -np.inf).all()
        assert np.array_equal(ref["album_groups"][0], ref["groups"][[0, 2, 6, 10]].sum(axis=0))
        k = 5
        per = 2                                                 # M/S pairs, or nchan = 2
        a = B.programme_needle(x[:per * k], lengths[:k], kind, limit_db=-12.0)
        b = B.programme_needle(np.ascontiguousarray(x[per * k:]), lengths[k:], kind, limit_db=-12.0)
        two = B.needle_albums(np.concatenate([a["hist"], b["hist"]]), np.concatenate([a["stats"], b["stats"]]), grp)
        for f in two:
            assert np.array_equal(np.asarray(two[f]).view(np.uint8), np.asarray(ref[f]).view(np.uint8)), f
    loud = B.programme_needle(x, lengths, O.PPM_MS, ms_gain_db=(0.0, 0.0))
    quiet = B.programme_needle(x, lengths, O.PPM_MS)
    live = lengths > 100
    assert (loud["peak"][live] > quiet["peak"][live]).all()
    c, s, rd = _private(x, lengths, O.PPM_MS, 2, 1024, 0.0, gains=(0.0, 0.0))
    assert np.array_equal(loud["hist"], c) and np.array_equal(u32(loud["reading"]), u32(rd))


def test_argument_errors():
    import meters_lv2_b200 as B
    g = B.NeedleMeters(3, O.PPM_IEC2)
    with pytest.raises(B.B200MError, match="histogram plane is off"):
        g.hist()
    with pytest.raises(B.B200MError, match="limit_db"):
        g.hist_enable(limit_db=np.nan)
    with pytest.raises(B.B200MError, match="histogram plane is off"):
        g.hist()
    L, E_INVAL = B.lib(), -1
    c = np.zeros((3, 242), np.uint64); s = np.zeros(3, B.PPM_HIST_STATS_DTYPE)
    g.hist_enable(limit_db=-np.inf)
    for args in ((g.h, None, s.ctypes.data_as(C.c_void_p), None), (g.h, c.ctypes.data_as(C.c_void_p), None, None),
                 (None, c.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), None)):
        assert L.b200m_ppm_hist_read(*args) == E_INVAL
    assert L.b200m_ppm_hist_enable(None, 1, 0.0, None) == E_INVAL
    assert L.b200m_ppm_hist_edges(None) == E_INVAL
    g.process(np.full((3, 17), 0.5, np.float32))
    c, s = g.hist()
    assert c.sum() == 3 * 4 and (s["over_groups"] == 4).all() and (s["overs"] == 1).all()   # -inf dB: L = 0, every reading over
    g.hist_enable(limit_db=np.inf)
    g.process(np.full((3, 16), 0.5, np.float32))
    assert not g.hist()[1]["over_groups"].any()
    with pytest.raises(B.B200MError, match="lengths"):
        B.programme_needle(np.zeros((2, 4), np.float32), [-1, 2], O.PPM_VU, nchan=1)
