"""GPU: the spectrum bank's long-term average spectrum plane (b200m_spec_ltas_*, Spectr30.ltas_enable / ltas) and
programme_spectrum, against the oracle of tests/_spec_ltas.py (the per-frame band power of the reference build's own filter
trajectory, summed in frame order)."""
import numpy as np
import pytest

import _signals as S
import _spec_ltas as L

pytestmark = pytest.mark.gpu


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _signal(rows, n, seed, fs=48000.0):
    x = S.white(rows, n, seed=seed)
    x[0] = 0.5 * S.sine(n, 1000.0, fs) + 0.01 * x[0]
    x[-1] *= np.float32(1e-4)                                # a quiet row: bands near the floor
    return x


def _same_ltas(tag, got, want):
    (gs, gc), (ws, wc) = got, want
    assert np.array_equal(gc, wc), (tag, np.argwhere(gc != wc)[:4])
    assert np.array_equal(u64(gs), u64(ws)), (tag, np.abs(gs - ws).max())


def _same_state(tag, banks, oracle, insts):
    for i in insts:
        oz, ov, om = oracle.state(i)
        for g in banks:
            z, v, m = g.state(i)
            assert np.array_equal(u64(z), u64(oz)) and np.array_equal(u32(v), u32(ov)) and np.array_equal(u32(m), u32(om)), (tag, i)


@pytest.mark.parametrize("rate,nchan,n_inst,blocks", [
    (48000.0, 2, 7, [1024] * 6 + [1, 8192, 3, 777, 64]),
    (48000.0, 1, 5, [1, 1, 2048, 8192, 100]),
    (22050.0, 2, 6, [1024, 8192, 1, 333]),
    (44100.0, 1, 9, [1024] * 3 + [8192, 1, 441]),
    (96000.0, 2, 3, [8192, 1, 4096, 7]),
    (192000.0, 2, 2, [8192, 8192, 1, 1920]),
])
def test_ltas_bit_exact_with_ports_unchanged(rate, nchan, n_inst, blocks):
    """sums and counts bit-identical to the oracle; the 60 ports and the filter states bit-identical with the plane on, off and in
    the reference build"""
    import torch
    import meters_lv2_b200 as B
    x = _signal(nchan * n_inst, sum(blocks), seed=600 + n_inst, fs=rate)
    on, off = B.Spectr30(n_inst, nchan, rate), B.Spectr30(n_inst, nchan, rate)
    on.ltas_enable()
    o = L.Spectr30(n_inst, nchan, rate)
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for b, n in enumerate(blocks):
        on.process(xd[:, pos:pos + n]); off.process(xd[:, pos:pos + n]); o.process(x[:, pos:pos + n], nthreads=4)
        pos += n
        p = o.read()
        assert np.array_equal(u32(on.read()), u32(p)) and np.array_equal(u32(off.read()), u32(p)), b
        if b % 3 == 2 or b == len(blocks) - 1:
            _same_ltas(b, on.ltas(), o.ltas())
    _same_state("end", (on, off), o, range(n_inst))
    s, c = on.ltas()
    counted = 30 if rate >= 44100 else 27
    # at 22.05 kHz the reference moves the top bands' upper edges below Nyquist (src/spectr.c:113-122) and the filters of bands
    # 27-29 diverge: their power is never finite, so they count no frame
    assert (c[:, :counted] == pos).all() and (s[:, :counted] > 0).all() and not c[:, counted:].any()


@pytest.mark.parametrize("nchan", [2, 1])
def test_ltas_non_finite_input(nchan):
    """NaN, +-Inf, denormals, zeros and clicks (host path): the counts skip the frames whose power is not finite, as the oracle's do,
    and the ports still equal the reference's"""
    import meters_lv2_b200 as B
    n_inst, blocks = 5, [1024, 1024, 1, 4096, 333, 1024]
    x = S.nasty(nchan * n_inst, sum(blocks), seed=610 + nchan)
    x[nchan, 1500] = np.float32(1e30)                        # finite input whose band power overflows float
    g = B.Spectr30(n_inst, nchan); g.ltas_enable()
    o = L.Spectr30(n_inst, nchan)
    pos = 0
    for n in blocks:
        blk = np.ascontiguousarray(x[:, pos:pos + n])
        g.process(blk); o.process(blk)
        pos += n
        assert np.array_equal(u32(g.read()), u32(o.read()))
        _same_ltas(pos, g.ltas(), o.ltas())
    s, c = g.ltas()
    assert (c < pos).any() and np.isfinite(s).all()
    _same_state("end", (g,), o, range(n_inst))


def test_ltas_ragged_paths_clear_and_enable():
    """ragged blocks (lengths 0 included) against private oracle instances fed only their own frames; the host path, the device path
    on a caller stream and switches between them; clear(inst) zeroes that row only (a fresh instance, also for the LTAS); enabling
    again zeroes every row; reading while the plane is off raises and the ports carry on"""
    import torch
    import meters_lv2_b200 as B
    n, nchan = 10, 2
    rng = np.random.default_rng(620)
    sizes = [1024, 512, 8192, 1, 1024, 700, 1024, 2048, 64, 1024]
    x = _signal(nchan * n, sum(sizes), seed=621)
    g = B.Spectr30(n, nchan)
    st = torch.cuda.Stream()
    g.ltas_enable(stream=st)
    priv = [L.Spectr30(1, nchan) for _ in range(n)]
    spd = np.full(n, 1.0, np.float32); rst = np.full(n, -4.0, np.float32)

    def want():
        s = np.concatenate([p.ltas()[0] for p in priv]); c = np.concatenate([p.ltas()[1] for p in priv])
        return s, c

    pos = 0
    for b, nf in enumerate(sizes):
        ln = rng.integers(0, nf + 1, size=n)
        ln[b % n] = 0
        ln[(b + 3) % n] = nf
        blk = x[:, pos:pos + nf]
        host = b % 3 == 1
        if host:
            g.process(np.ascontiguousarray(blk), speed=spd, reset=rst, lengths=ln)
        else:
            with torch.cuda.stream(st):
                xd = torch.from_numpy(np.ascontiguousarray(blk)).cuda()
            g.process(xd, speed=spd, reset=rst, lengths=ln, stream=st)
        for i in range(n):
            if ln[i]:
                priv[i].process(blk[nchan * i:nchan * (i + 1), :ln[i]])
        pos += nf
        rs = None if host else st
        _same_ltas(b, g.ltas(stream=rs), want())
        got = g.read(stream=rs)
        for i in range(n):
            assert np.array_equal(u32(got[i]), u32(priv[i].read()[0])), (b, i)
        if b == 4:
            before = g.ltas(stream=rs)
            g.clear(3, stream=rs)
            priv[3] = L.Spectr30(1, nchan)
            after = g.ltas(stream=rs)
            assert (after[0][3] == 0).all() and (after[1][3] == 0).all()
            keep = np.arange(n) != 3
            assert np.array_equal(u64(after[0][keep]), u64(before[0][keep])) and np.array_equal(after[1][keep], before[1][keep])
        if b == 6:
            g.ltas_enable(stream=rs)
            s, c = g.ltas(stream=rs)
            assert not s.any() and not c.any()
            for p in priv:
                p.clear_ltas()
    z, v, m = g.state(3, stream=st); oz, ov, om = priv[3].state(0)
    assert np.array_equal(u64(z), u64(oz)) and np.array_equal(u32(v), u32(ov))
    g.ltas_enable(False, stream=st)
    with pytest.raises(B.B200MError, match="LTAS plane is off"):
        g.ltas(stream=st)
    blk = np.ascontiguousarray(x[:, :256])
    g.process(blk, speed=spd, reset=rst, lengths=np.full(n, 256))
    for i in range(n):
        priv[i].process(blk[nchan * i:nchan * (i + 1)])
        assert np.array_equal(u32(g.read()[i]), u32(priv[i].read()[0])), i


@pytest.mark.parametrize("band,amp", [(16, 0.5), (6, 0.25), (26, 0.9)])
def test_ltas_of_a_sine_at_a_band_centre(band, amp):
    """a settled sine of amplitude A at a band's nominal centre: that band's ltas_db is 20 log10 A within 0.01 dB (the band-pass
    gain at the nominal centre is 1 within 1e-10 dB at 48 kHz; the rest is the partial period at the ends and float32 power), and
    within 0.1 dB of the band's settled level port"""
    import torch
    import meters_lv2_b200 as B
    fs, nf = 48000.0, 1024
    f = float(B.SPEC_BAND_HZ[band])
    n = 4 * 48 * nf
    x = S.sine(n, f, fs, amp=amp)[None, :]
    g = B.Spectr30(1, 1); g.ltas_enable()
    xd = torch.from_numpy(x).cuda()
    for k in range(n // nf):
        if k == 48:                                          # 1 s to settle, then 3 s averaged
            g.ltas_enable()
        g.process(xd[:, k * nf:(k + 1) * nf])
    s, c = g.ltas()
    db = B._ltas_db(B._ltas(s, c))[0]
    want = 20 * np.log10(amp)
    assert abs(db[band] - want) <= 0.01, (db[band], want)
    port = float(g.read()[0, band])
    assert abs(db[band] - port) <= 0.1, (db[band], port)
    others = np.delete(db, [band - 1, band, band + 1])
    assert (others < want - 20).all()                       # the neighbours' skirts aside, the tone stays in its band


def _clips(n, nchan, lengths, seed):
    x = S.white(n * nchan, int(max(lengths)) + 5, seed=seed)
    for i in range(n):
        x[i * nchan:(i + 1) * nchan] *= np.float32(10.0 ** (-(i % 7) / 4))
        x[i * nchan:(i + 1) * nchan, lengths[i]:] = np.nan   # past a clip's end: never read into a result
    return x


def _private(x, lengths, nchan, block, speed, rate=48000.0):
    """each clip fed alone to an oracle instance in `block`-frame pieces, the reset port held as programme_spectrum holds it"""
    rst = -4.0 if np.float32(speed) == 1.0 else 0.0
    s, c, pk = [], [], []
    for i, ln in enumerate(lengths):
        o = L.Spectr30(1, nchan, rate)
        for off in range(0, int(ln), block):
            o.process(x[i * nchan:(i + 1) * nchan, off:min(off + block, ln)], speed, rst)
        a, b = o.ltas()
        s.append(a[0]); c.append(b[0])
        pk.append(o.read()[0, 30:] if ln else np.full(30, -100.0, np.float32))
    return np.array(s), np.array(c), np.array(pk, np.float32)


@pytest.mark.parametrize("nchan,block,speed", [(2, 1024, 1.0), (1, 777, 2.5)])
def test_programme_spectrum_equals_private_instances(nchan, block, speed):
    import meters_lv2_b200 as B
    lengths = np.array([4000, 0, 1024, 1, 9000, 777, 2 * 777, 12345, 50])
    n = lengths.size
    x = _clips(n, nchan, lengths, seed=630 + nchan)
    r = B.programme_spectrum(x, lengths, nchan=nchan, speed=speed, block=block)
    s, c, pk = _private(x, lengths, nchan, block, speed)
    assert np.array_equal(u64(r["sums"]), u64(s)) and np.array_equal(r["counts"], c)
    assert r["counts"].dtype == np.int64 and r["ltas"].dtype == np.float64 and r["peak_db"].dtype == np.float32
    assert np.array_equal(u32(r["peak_db"]), u32(pk)) and (r["peak_db"] > -500).all()
    assert np.array_equal(np.isnan(r["ltas"]), c == 0)
    assert np.array_equal(u64(r["ltas"][c > 0]), u64(s[c > 0] / c[c > 0]))
    assert np.isnan(r["ltas"][1]).all() and (r["ltas_db"][1] == -100).all() and (r["peak_db"][1] == -100).all() and (r["counts"][1] == 0).all()
    assert np.array_equal(r["ltas_db"], B._ltas_db(r["ltas"]))
    assert (r["counts"] == lengths[:, None]).all()


def test_programme_spectrum_inputs_albums_and_shards():
    """numpy, CPU-tensor, CUDA-tensor and callable inputs give the same bits; albums with unassigned clips and empty albums are
    spectrum_albums of the clip rows; two shards' rows pooled give the one bank's album values bit for bit"""
    import torch
    import meters_lv2_b200 as B
    lengths = np.array([3000, 5000, 0, 1024, 4097, 10, 2048, 6000, 333, 4500, 1])
    n, nchan = lengths.size, 2
    x = _clips(n, nchan, lengths, seed=640)
    grp = np.array([0, 2, 0, -1, 2, 4, 0, -1, 2, 4, 0])       # albums 1 and 3 have no members
    ref = B.programme_spectrum(x, lengths, groups=grp)
    xd = torch.from_numpy(x).cuda()
    for tag, inp in (("cpu tensor", torch.from_numpy(x)), ("cuda", xd), ("callable", lambda off, nf: xd[:, off:off + nf])):
        r = B.programme_spectrum(inp, lengths, groups=grp)
        assert set(r) == set(ref), tag
        for k in ref:
            assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(ref[k]).view(np.uint8)), (tag, k)
    alb = B.spectrum_albums(ref["sums"], ref["counts"], ref["peak_db"], grp)
    for k in alb:
        assert np.array_equal(np.asarray(ref[k]).view(np.uint8), np.asarray(alb[k]).view(np.uint8)), k
    assert list(ref["album_n_clips"]) == [4, 0, 3, 0, 2]
    assert np.isnan(ref["album_ltas"][[1, 3]]).all() and (ref["album_ltas_db"][[1, 3]] == -100).all() and (ref["album_peak_db"][[1, 3]] == -100).all()
    # album 0 holds the empty clip 2: it adds no frames
    assert (ref["counts"][[0, 6, 10]].sum(axis=0) == lengths[[0, 6, 10]].sum()).all()
    k = 5
    a = B.programme_spectrum(x[:k * nchan], lengths[:k])
    b = B.programme_spectrum(np.ascontiguousarray(x[k * nchan:]), lengths[k:])
    two = B.spectrum_albums(*(np.concatenate([a[f], b[f]]) for f in ("sums", "counts", "peak_db")), grp)
    for f in two:
        assert np.array_equal(np.asarray(two[f]).view(np.uint8), np.asarray(ref[f]).view(np.uint8)), f


def test_programme_spectrum_tolerance_mode():
    """B200M_PREC_FMA: ltas_db within 1e-4 dB of exact mode and the same counts, non-finite input included"""
    import meters_lv2_b200 as B
    lengths = np.array([20000, 7000, 1, 15000, 0, 9000])
    n, nchan = lengths.size, 2
    x = _clips(n, nchan, lengths, seed=650)
    x[6, 3000] = np.nan; x[1, 100] = np.inf
    ex = B.programme_spectrum(x, lengths, precision=B.PREC_EXACT)
    fm = B.programme_spectrum(x, lengths, precision=B.PREC_FMA)
    assert np.array_equal(ex["counts"], fm["counts"])
    live = ex["ltas_db"] > -100
    assert np.array_equal(live, fm["ltas_db"] > -100)
    assert np.abs(ex["ltas_db"][live] - fm["ltas_db"][live]).max() <= 1e-4
    assert np.abs(ex["peak_db"].astype(np.float64) - fm["peak_db"]).max() <= 1e-4
