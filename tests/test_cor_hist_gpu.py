"""GPU: the correlation bank's histogram plane (b200m_cor_hist_*, Stcorrdsp.hist_enable / hist) and programme_correlation, against
the oracle of tests/_cor_hist.py (the per-frame readings of the reference build's own trajectory, counted and summed in frame
order)."""
import ctypes as C

import numpy as np
import pytest

import _cor_hist as H
import _signals as S
from test_cor_hist_cpu import stereo

pytestmark = pytest.mark.gpu


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _same_hist(tag, got, want):
    (gc, gs), (wc, ws) = got, want
    assert np.array_equal(gc, wc), (tag, np.argwhere(gc != wc)[:4])
    assert np.array_equal(u64(gs), u64(ws)), (tag, np.abs(gs - ws).max())


def _same_bank(tag, a, b, stream=None):
    """readings and the five states of two banks bit for bit"""
    assert np.array_equal(u32(a.read(stream)), u32(b.read(stream))), tag
    assert np.array_equal(u32(a.state(stream)), u32(b.state(stream))), tag


@pytest.mark.parametrize("rate,tcf,n,blocks", [
    (48000, 0.3, 37, [1024] * 6 + [1, 8192, 3, 777, 64]),
    (48000, 1.0, 5, [1, 1, 2048, 8192, 100]),
    (22050, 0.3, 6, [1024, 8192, 1, 333]),
    (44100, 0.3, 9, [1024] * 3 + [8192, 1, 441]),
    (88200, 0.3, 4, [8192, 1024, 5]),
    (96000, 0.3, 3, [8192, 1, 4096, 7]),
    (176400, 0.3, 2, [8192, 8192, 19]),
    (192000, 0.3, 2, [8192, 8192, 1, 1920]),
])
def test_hist_bit_exact_with_ports_unchanged(rate, tcf, n, blocks):
    """counts and sums bit-identical to the oracle after every block; readings and states bit-identical with the plane on, off and
    in the reference build"""
    import torch
    import meters_lv2_b200 as B
    x = stereo(n, sum(blocks), seed=800 + n)
    on, off = B.Stcorrdsp(n, rate, tcf=tcf), B.Stcorrdsp(n, rate, tcf=tcf)
    on.hist_enable()
    o = H.Stcorr(n, rate, tcf=tcf)
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for b, nf in enumerate(blocks):
        on.process(xd[:, pos:pos + nf]); off.process(xd[:, pos:pos + nf]); o.process(x[:, pos:pos + nf])
        pos += nf
        p = o.read()
        assert np.array_equal(u32(on.read()), u32(p)) and np.array_equal(u32(off.read()), u32(p)), b
        _same_hist(b, on.hist(), o.hist())
    _same_bank("end", on, off)
    assert np.array_equal(u32(on.state()), u32(o.peek()))
    c, _ = on.hist()
    assert (c[:n - 1].sum(axis=1) > 0.9 * pos).all() and c[n - 1].sum() == 0      # the quiet pair stays under the gate


def test_tolerance_mode_with_the_plane_runs_exact():
    """B200M_PREC_FMA with the plane on gives the exact-mode plane, states and readings bit for bit; with the plane off (also after
    enabling and disabling it) tolerance mode still runs its time-parallel kernel, whose bits differ from exact mode's"""
    import torch
    import meters_lv2_b200 as B
    n, blocks = 16, [1024] * 12 + [333, 8192]
    x = stereo(n, sum(blocks), seed=810)
    xd = torch.from_numpy(x).cuda()
    ex, fh, fm, ft = (B.Stcorrdsp(n) for _ in range(4))
    for g in (fh, fm, ft):
        g.set_precision(B.PREC_FMA)
    ex.hist_enable(); fh.hist_enable()
    ft.hist_enable(); ft.hist_enable(False)
    differ = False
    pos = 0
    for nf in blocks:
        for g in (ex, fh, fm, ft):
            g.process(xd[:, pos:pos + nf])
        pos += nf
        _same_bank(pos, ex, fh)
        _same_hist(pos, fh.hist(), ex.hist())
        _same_bank(pos, fm, ft)
        differ |= not np.array_equal(u32(fm.state()), u32(ex.state()))
        assert np.abs(fm.read() - ex.read()).max() <= 1e-5
    assert differ


def test_hist_non_finite_input():
    """NaN, +-Inf, denormals, zeros and clicks (host path): a non-finite state leaves its block's remaining frames uncounted, as in the
    oracle, and the readings still equal the reference's"""
    import meters_lv2_b200 as B
    n, blocks = 5, [1024, 1024, 1, 4096, 333, 1024]
    x = S.nasty(2 * n, sum(blocks), seed=820)
    x[2, 1500] = np.float32(1e30)                             # finite input whose power overflows float
    for gate_db in (-70.0, -np.inf):
        g = B.Stcorrdsp(n); g.hist_enable(gate_db=gate_db)
        o = H.Stcorr(n, gate_db=gate_db)
        pos = 0
        for nf in blocks:
            blk = np.ascontiguousarray(x[:, pos:pos + nf])
            g.process(blk); o.process(blk)
            pos += nf
            assert np.array_equal(u32(g.read()), u32(o.read()))
            _same_hist(pos, g.hist(), o.hist())
        c, s = g.hist()
        assert (c.sum(axis=1) < pos).any() and np.isfinite(s).all()


def test_hist_ragged_holds_paths_clear_and_enable():
    """ragged blocks (lengths 0 included) and process_ctl holds against private oracle pairs fed only their own frames; the host path,
    the device path on a caller stream and switches between them; clear(inst) zeroes that row only, clear() every row; disabling
    stops counting and keeps the ports going, enabling again zeroes every row"""
    import torch
    import meters_lv2_b200 as B
    n = 11
    rng = np.random.default_rng(830)
    sizes = [1024, 512, 8192, 1, 1024, 700, 1024, 2048, 64, 1024, 1024, 300]
    x = stereo(n, sum(sizes), seed=831)
    g = B.Stcorrdsp(n)
    st = torch.cuda.Stream()
    g.hist_enable(stream=st)
    priv = [H.Stcorr(1) for _ in range(n)]
    counting = True

    def want():
        return np.concatenate([p.hist()[0] for p in priv]), np.concatenate([p.hist()[1] for p in priv])

    pos = 0
    for b, nf in enumerate(sizes):
        ln = rng.integers(0, nf + 1, size=n)
        ln[b % n] = 0
        ln[(b + 3) % n] = nf
        ctl = b % 4 == 3                                       # a process_ctl block: held pairs, the others run nf frames
        if ctl:
            run = (ln > 0).astype(np.uint8)
            ln = np.where(run, nf, 0)
        blk = x[:, pos:pos + nf]
        host = b % 3 == 1
        kw = dict(run=run) if ctl else dict(lengths=ln)
        if host:
            g.process(np.ascontiguousarray(blk), **kw)
        else:
            with torch.cuda.stream(st):
                xd = torch.from_numpy(np.ascontiguousarray(blk)).cuda()
            g.process(xd, stream=st, **kw)
        before = [p.hist() for p in priv]
        for i in range(n):
            if ln[i]:
                priv[i].process(blk[2 * i:2 * i + 2, :ln[i]])
        if not counting:                                       # the plane is off: the private oracles' counts stay put
            for p, (c0, s0) in zip(priv, before):
                p.counts[:] = c0; p.sums[:] = s0
        pos += nf
        rs = None if host else st
        if counting:
            _same_hist(b, g.hist(stream=rs), want())
        got = g.read(stream=rs)
        for i in range(n):
            assert np.array_equal(u32(got[i]), u32(priv[i].read()[0])), (b, i)
        if b == 4:
            before = g.hist(stream=rs)
            g.clear(3, stream=rs)
            priv[3] = H.Stcorr(1)
            after = g.hist(stream=rs)
            assert not after[0][3].any() and after[1][3] == 0
            keep = np.arange(n) != 3
            assert np.array_equal(after[0][keep], before[0][keep]) and np.array_equal(u64(after[1][keep]), u64(before[1][keep]))
        if b == 6:
            g.clear(stream=rs)
            priv = [H.Stcorr(1) for _ in range(n)]
            c, s = g.hist(stream=rs)
            assert not c.any() and not s.any()
        if b == 7:
            g.hist_enable(False, stream=rs)
            counting = False
            with pytest.raises(B.B200MError, match="histogram plane is off"):
                g.hist(stream=rs)
        if b == 9:
            g.hist_enable(gate_db=-np.inf, stream=rs)
            counting = True
            for p in priv:
                p.clear_hist(-np.inf)
            c, s = g.hist(stream=rs)
            assert not c.any() and not s.any()
    assert np.array_equal(u32(g.state(stream=st)), u32(np.concatenate([p.peek() for p in priv])))


@pytest.mark.parametrize("ragged", [False, True])
def test_phasewheel_fed_bank_counts_like_a_plain_bank(ragged):
    """a bank attached to a phasewheel bank (the fused ring feed, and its unfused ragged feed) gives the same plane, readings and
    states as an unattached bank fed the same blocks"""
    import torch
    import meters_lv2_b200 as B
    n, blocks = 40, [1024] * 5 + [512, 8192, 77]
    rng = np.random.default_rng(840)
    x = stereo(n, sum(blocks), seed=841)
    xd = torch.from_numpy(x).cuda()
    pw, fed, plain = B.Phasewheel(n, 1024), B.Stcorrdsp(n), B.Stcorrdsp(n)
    pw.attach_cor(fed)
    fed.hist_enable(); plain.hist_enable()
    pos = 0
    for nf in blocks:
        ln = rng.integers(0, nf + 1, size=n) if ragged else None
        pw.process(xd[:, pos:pos + nf], lengths=ln)
        plain.process(xd[:, pos:pos + nf], lengths=ln)
        pos += nf
        _same_hist(pos, fed.hist(), plain.hist())
        _same_bank(pos, fed, plain)
    assert fed.hist()[0].sum() > 0
    pw.attach_cor(None)


def test_known_answers():
    """after 1 s of warm-up (the reading's sqrt (zll * zrr + 1e-10) holds it near 0 while the filters are quiet): identical channels
    count every frame in bin 199, inverted channels in bin 0 (below0 == 1); independent noise has |mean| < 0.05 over 10 s; noise at
    -80 dBFS RMS under the default -70 dB gate counts no frame"""
    import torch
    import meters_lv2_b200 as B
    nf, block = 480 * 1024, 1024
    a = S.white(1, nf, seed=850)[0]
    w = [S.white(1, nf, seed=851 + k)[0] for k in range(3)]
    q = np.float32(1e-4 * np.sqrt(3.0) / 0.5)                 # white()'s channel 0 is uniform (-0.5, 0.5)
    x = np.ascontiguousarray(np.stack([a, a, a, -a, a, w[0], w[1] * q, w[2] * q]), np.float32)
    g = B.Stcorrdsp(4)
    xd = torch.from_numpy(x).cuda()
    for k in range(nf // block):
        if k == 48:
            g.hist_enable()
        g.process(xd[:, k * block:(k + 1) * block])
    c, s = g.hist()
    d = B._cor_dist(c, s)
    assert c[0, 199] == c[0].sum() == nf - 48 * block
    assert c[1, 0] == c[1].sum() == nf - 48 * block and d["below0"][1] == 1.0 and d["p1"][1] == -1.0
    assert c[2].sum() == nf - 48 * block and abs(d["mean"][2]) < 0.05
    assert c[3].sum() == 0 and np.isnan(d["mean"][3])


def _clips(n, lengths, seed):
    x = stereo(n, int(max(lengths)) + 5, seed=seed)
    for i in range(n):
        x[2 * i:2 * i + 2, lengths[i]:] = np.nan               # past a clip's end: never read into a result
    return x


def _private(x, lengths, block, gate_db=-70.0, rate=48000, tcf=0.3):
    """each clip fed alone to an oracle pair in `block`-frame pieces"""
    c, s, rd = [], [], []
    for i, ln in enumerate(lengths):
        o = H.Stcorr(1, rate, tcf=tcf, gate_db=gate_db)
        for off in range(0, int(ln), block):
            o.process(x[2 * i:2 * i + 2, off:min(off + block, ln)])
        a, b = o.hist()
        c.append(a[0]); s.append(b[0]); rd.append(o.read()[0])
    return np.array(c), np.array(s), np.array(rd, np.float32)


@pytest.mark.parametrize("block,gate_db,tcf", [(1024, -70.0, 0.3), (777, -np.inf, 1.0)])
def test_programme_correlation_equals_private_pairs(block, gate_db, tcf):
    import meters_lv2_b200 as B
    lengths = np.array([40000, 0, 1024, 1, 90000, 777, 2 * 777, 12345, 50])
    n = lengths.size
    x = _clips(n, lengths, seed=860)
    r = B.programme_correlation(x, lengths, tcf=tcf, gate_db=gate_db, block=block)
    c, s, rd = _private(x, lengths, block, gate_db, tcf=tcf)
    assert np.array_equal(r["hist"], c) and np.array_equal(u64(r["sums"]), u64(s)) and np.array_equal(u32(r["reading"]), u32(rd))
    assert r["hist"].dtype == np.int64 and r["frames"].dtype == np.int64 and r["reading"].dtype == np.float32
    d = B._cor_dist(c, s)
    for k in d:
        assert np.array_equal(r[k], d[k], equal_nan=True), k
    assert r["frames"][1] == 0 and r["reading"][1] == 0 and all(np.isnan(r[k][1]) for k in ("mean", "below0", "p1", "p5"))
    if gate_db == -np.inf:
        assert np.array_equal(r["frames"], lengths)


def test_programme_correlation_inputs_albums_and_shards():
    """numpy, CUDA-tensor and callable inputs give the same bits; albums with unassigned clips and empty albums are
    correlation_albums of the clip rows; two banks' rows pooled give the one bank's album values bit for bit"""
    import torch
    import meters_lv2_b200 as B
    lengths = np.array([3000, 50000, 0, 1024, 4097, 10, 20480, 6000, 333, 4500, 1])
    n = lengths.size
    x = _clips(n, lengths, seed=870)
    grp = np.array([0, 2, 0, -1, 2, 4, 0, -1, 2, 4, 0])        # albums 1 and 3 have no members
    ref = B.programme_correlation(x, lengths, groups=grp)
    xd = torch.from_numpy(x).cuda()
    for tag, inp in (("cuda", xd), ("callable", lambda off, nf: xd[:, off:off + nf])):
        r = B.programme_correlation(inp, lengths, groups=grp)
        assert set(r) == set(ref), tag
        for k in ref:
            assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(ref[k]).view(np.uint8)), (tag, k)
    alb = B.correlation_albums(ref["hist"], ref["sums"], grp)
    for k in alb:
        assert np.array_equal(np.asarray(ref[k]).view(np.uint8), np.asarray(alb[k]).view(np.uint8)), k
    assert list(ref["album_n_clips"]) == [4, 0, 3, 0, 2]
    assert list(ref["album_frames"][[1, 3]]) == [0, 0] and np.isnan(ref["album_mean"][[1, 3]]).all()
    assert np.array_equal(ref["album_frames"][0], ref["frames"][[0, 2, 6, 10]].sum())
    k = 5
    a = B.programme_correlation(x[:2 * k], lengths[:k])
    b = B.programme_correlation(np.ascontiguousarray(x[2 * k:]), lengths[k:])
    two = B.correlation_albums(np.concatenate([a["hist"], b["hist"]]), np.concatenate([a["sums"], b["sums"]]), grp)
    for f in two:
        assert np.array_equal(np.asarray(two[f]).view(np.uint8), np.asarray(ref[f]).view(np.uint8)), f


def test_argument_errors():
    import meters_lv2_b200 as B
    g = B.Stcorrdsp(3)
    with pytest.raises(B.B200MError, match="histogram plane is off"):
        g.hist()
    for bad in (np.nan, np.inf):
        with pytest.raises(B.B200MError, match="gate_db"):
            g.hist_enable(gate_db=bad)
    with pytest.raises(B.B200MError, match="histogram plane is off"):
        g.hist()
    g.hist_enable(gate_db=-np.inf)
    L, E_INVAL = B.lib(), -1
    c = np.zeros((3, 200), np.uint64); s = np.zeros(3)
    for args in ((g.h, None, s.ctypes.data_as(C.c_void_p), None), (g.h, c.ctypes.data_as(C.c_void_p), None, None),
                 (None, c.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), None)):
        assert L.b200m_cor_hist_read(*args) == E_INVAL
    assert L.b200m_cor_hist_enable(None, 1, -70.0, None) == E_INVAL
    g.process(np.zeros((6, 16), np.float32))
    assert g.hist()[0].sum() == 3 * 16
