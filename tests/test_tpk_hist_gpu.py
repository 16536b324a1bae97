"""The true-peak / K-meter bank's histogram plane (b200m_tpk_hist_*) against its oracle (tests/_tpk_hist.py): bit-exact counts and
statistics after every block, ports and states unchanged by the plane, the FMA bank, non-finite input, ragged blocks, caller
streams, clear / reset / read, enable and limits, the refused calls, known answers and programme_truepeak."""
import ctypes as C

import numpy as np
import pytest

import _tpk_hist as H

pytestmark = pytest.mark.gpu

RATES = (22050.0, 44100.0, 48000.0, 88200.0, 96000.0, 176400.0, 192000.0)
TPKM, TPO, KMO = 3, 1, 2
E_INVAL, E_UNSUPPORTED = -1, -4              # B200M_E_INVAL, B200M_E_UNSUPPORTED


def B():
    import meters_lv2_b200 as b
    return b


def _programme(n, nframes, seed, loud=3.0):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, nframes)) * rng.uniform(0.05, 1.0, (n, 1))).astype(np.float32)
    x[:, nframes // 3: nframes // 2] *= loud
    return x


def _same(bank_hist, oracle_hist):
    for u, v in zip(bank_hist, oracle_hist):
        if u is None or v is None:
            assert u is None and v is None
        elif u.dtype == np.int64:
            assert np.array_equal(u, v)
        else:
            assert u.tobytes() == v.tobytes()


def _state_bits(bank):
    st = bank.state()
    return b"".join(np.ascontiguousarray(st[k]).tobytes() for k in ("m", "p", "z1", "z2", "res", "km"))


def _run(flags, fs, n=20, nframes=3000, block=1024, lengths=None, device_path=False, tp_db=-1.0, km_db=-30.0):
    import torch
    b = B()
    x = _programme(n, nframes, int(fs) + flags)
    bank = b.TruePeakKmeter(n, fs, flags)
    plain = b.TruePeakKmeter(n, fs, flags)
    o = H.TpkHist(n, fs, flags, tp_db, km_db)
    bank.hist_enable(tp_limit_db=tp_db, km_limit_db=km_db)
    for off in range(0, nframes, block):
        xb = np.ascontiguousarray(x[:, off:off + block])
        lb = None if lengths is None else np.clip(np.asarray(lengths) - off, 0, xb.shape[1])
        xin = torch.from_numpy(xb).cuda() if device_path else xb
        bank.process(xin, lengths=lb)
        plain.process(xin, lengths=lb)
        o.process(xb, lb)
        r1, r0 = bank.read(), plain.read()
        assert r1.tobytes() == r0.tobytes()
        _same(bank.hist(), o.hist())
    assert _state_bits(bank) == _state_bits(plain)
    return bank, o


@pytest.mark.parametrize("fs", RATES)
@pytest.mark.parametrize("flags", (TPKM, TPO, KMO))
def test_counts_match_oracle_every_block(fs, flags):
    _run(flags, fs)


def test_fma_bank_with_plane_equals_exact():
    b = B()
    x = _programme(24, 2048, 5)
    ex, fm = b.TruePeakKmeter(24), b.TruePeakKmeter(24)
    fm.set_precision(b.PREC_FMA)
    for k in (ex, fm):
        k.hist_enable()
    for off in (0, 1024):
        xb = np.ascontiguousarray(x[:, off:off + 1024])
        ex.process(xb); fm.process(xb)
        assert ex.read().tobytes() == fm.read().tobytes()
    _same(ex.hist(), fm.hist())
    assert _state_bits(ex) == _state_bits(fm)


def test_nonfinite_input():
    b = B()
    x = _programme(16, 2048, 9) * 0.2
    x[0, 300] = np.nan; x[1, 700] = np.inf; x[2, 1500] = -np.inf; x[3, 40:80] = np.float32(1e-40)
    bank = b.TruePeakKmeter(16); o = H.TpkHist(16)
    bank.hist_enable()
    for off in (0, 1024):
        xb = np.ascontiguousarray(x[:, off:off + 1024])
        bank.process(xb); o.process(xb, read=False)
    h = bank.hist()
    _same(h, o.hist())
    assert h[1]["nonfinite"][0] > 0 and h[1]["nonfinite"][1] > 0 and h[3]["nonfinite"][0] > 0


def test_ragged_blocks_with_holds_and_tails():
    n = 33
    rng = np.random.default_rng(1)
    lengths = rng.integers(0, 3000, n); lengths[:4] = (0, 1, 2999, 1023)
    for flags in (TPKM, TPO, KMO):
        _run(flags, 48000.0, n=n, nframes=3000, block=1000, lengths=lengths, km_db=-20.0)
        # blocks with nfram mod 4 tails, runs continuing across them
        _run(flags, 44100.0, n=n, nframes=2003, block=501, lengths=np.minimum(lengths, 2003))


def test_device_path_on_a_caller_stream():
    import torch
    b = B()
    x = _programme(16, 2048, 4)
    bank = b.TruePeakKmeter(16); o = H.TpkHist(16)
    s = torch.cuda.Stream()
    bank.hist_enable(stream=s)
    with torch.cuda.stream(s):
        for off in (0, 1024):
            xb = np.ascontiguousarray(x[:, off:off + 1024])
            bank.process(torch.from_numpy(xb).cuda(), stream=s)
            o.process(xb, read=False)
    _same(bank.hist(stream=s), o.hist())
    _run(TPKM, 48000.0, n=16, nframes=2048, device_path=True)


def test_clear_reset_read_and_reenable():
    b = B()
    x = _programme(16, 2048, 8)
    bank = b.TruePeakKmeter(16); o = H.TpkHist(16)
    bank.hist_enable()
    bank.process(x[:, :1024]); o.process(x[:, :1024], read=False)
    bank.clear(5); o.clear(5)
    _same(bank.hist(), o.hist())
    bank.reset(); bank.read(); b.lib().b200m_tpk_reset_kmeter(bank.h, None)
    o.reset()
    _same(bank.hist(), o.hist())                                   # reset, reset_kmeter and read leave the plane alone
    bank.process(np.ascontiguousarray(x[:, 1024:])); o.process(np.ascontiguousarray(x[:, 1024:]), read=False)
    _same(bank.hist(), o.hist())
    bank.hist_enable(False)
    bank.process(x[:, :1024])                                       # off: nothing counts, and the rows cannot be read
    o.process(x[:, :1024], read=False)                              # (the meters run on; the re-enable below empties the rows)
    with pytest.raises(b.B200MError):
        bank.hist()
    bank.hist_enable(tp_limit_db=-6.0, km_limit_db=-40.0)          # re-enable: empty rows, new limits
    o.clear_hist(-6.0, -40.0)
    bank.process(x[:, 1024:]); o.process(np.ascontiguousarray(x[:, 1024:]), read=False)
    _same(bank.hist(), o.hist())
    for lim in ((np.inf, -np.inf), (-np.inf, np.inf)):
        bank.hist_enable(tp_limit_db=lim[0], km_limit_db=lim[1]); o.clear_hist(*lim)
        bank.process(x[:, :1024]); o.process(x[:, :1024], read=False)
        _same(bank.hist(), o.hist())


def test_refused_calls():
    b = B()
    bank = b.TruePeakKmeter(16, flags=TPO)
    with pytest.raises(b.B200MError):
        bank.hist_enable(tp_limit_db=float("nan"))
    bank.hist_enable()
    with pytest.raises(b.B200MError):
        bank.process_max(np.zeros((16, 256), np.float32))
    L = b.lib()
    c = np.zeros((16, 242), np.uint64); s = np.zeros(16, b.PPM_HIST_STATS_DTYPE)
    assert L.b200m_tpk_hist_read(bank.h, c.ctypes.data, s.ctypes.data, c.ctypes.data, s.ctypes.data, None) == E_INVAL
    assert L.b200m_tpk_hist_read(bank.h, None, None, None, None, None) == E_INVAL
    r = b.EBUr128(4)
    tp = L.b200m_r128_tpk(r.h)
    assert L.b200m_tpk_hist_enable(C.c_void_p(tp), 1, -1.0, -10.0, None) == E_UNSUPPORTED
    r.close()


def test_known_answers():
    b = B()
    fs, n, nf = 48000.0, 16, 48 * 1024
    A = 10.0 ** (-6.25 / 20.0)                                      # mid-bin: the FIR's passband ripple stays inside it
    t = np.arange(nf)
    x = np.tile((A * np.sin(np.pi / 2 * t + np.pi / 4)).astype(np.float32), (n, 1))     # fs/4, 45 degrees: samples of A/sqrt(2)
    assert np.all(np.abs(np.abs(x) - np.float32(A / np.sqrt(2))) <= 1e-7)
    bank = b.TruePeakKmeter(n, fs); bank.hist_enable()
    for off in range(0, nf, 1024):
        bank.process(np.ascontiguousarray(x[:, off:off + 1024]))
    tc, ts, kc, ks = bank.hist()
    edges = np.asarray(b.PPM_HIST_EDGES)
    k = int(np.searchsorted(edges, np.float32(A), side="right"))
    # the 4x-oversampled frames of this sine alternate: every other one holds a crest (A), the others peak at 45 degrees from it
    # (A / sqrt 2, the sample peak); after the FIR settles the crest frames sit in the bin of 20 log10 A, 3 dB above the sample peak
    k2 = int(np.searchsorted(edges, np.float32(A / np.sqrt(2)), side="right"))
    assert (tc[:, k] >= nf // 2 - 64).all() and (tc[:, k] + tc[:, k2] >= nf - 64).all()
    assert (np.searchsorted(edges, ts["peak"], side="right") == k).all()
    assert (np.argmax(kc, axis=1) == k).all()                       # the settled K-meter reads A (sine-calibrated)
    assert (kc[:, k] > nf // 4 // 2).all()


def test_programme_truepeak_against_private_banks():
    import torch
    b = B()
    n, per = 5, 2
    lengths = np.array([3000, 1700, 0, 2500, 999])
    x = _programme(n * per, 3000, 21)
    grp = np.array([0, 1, 0, -1, 1])
    res = {}
    for kind in ("numpy", "cuda", "callable"):
        xin = x if kind == "numpy" else torch.from_numpy(x).cuda() if kind == "cuda" else (lambda off, nf: x[:, off:off + nf])
        res[kind] = b.programme_truepeak(xin, lengths, nchan=per, block=1000, groups=grp)
    for k, v in res["numpy"].items():
        for kind in ("cuda", "callable"):
            assert np.asarray(v).tobytes() == np.asarray(res[kind][k]).tobytes(), k
    out = res["numpy"]
    for i in range(n):
        bank = b.TruePeakKmeter(per); bank.hist_enable(True, -1.0, -10.0)
        for off in range(0, int(lengths[i]), 1000):
            bank.process(np.ascontiguousarray(x[i * per:(i + 1) * per, off:min(off + 1000, int(lengths[i]))]))
        tc, ts, kc, ks = bank.hist()
        assert np.array_equal(out["tp_hist"][i], tc) and np.array_equal(out["km_hist"][i], kc)
        assert out["tp_stats"][i].tobytes() == ts.tobytes() and out["km_stats"][i].tobytes() == ks.tobytes()
        if lengths[i]:
            r = bank.read()
            assert out["tp_p"][i].tobytes() == r["tp_p"].tobytes() and out["tp_m"][i].tobytes() == r["tp_m"].tobytes()
            assert out["km_rms"][i].tobytes() == r["km_rms"].tobytes() and out["km_peak"][i].tobytes() == r["km_peak"].tobytes()
    # two shards pool to one bank's albums
    a = b.programme_truepeak(x[:6], lengths[:3], nchan=per, block=1000)
    c = b.programme_truepeak(x[6:], lengths[3:], nchan=per, block=1000)
    pooled = b.needle_albums(np.concatenate([a["tp_hist"], c["tp_hist"]]), np.concatenate([a["tp_stats"], c["tp_stats"]]), grp)
    for k, v in pooled.items():
        assert v.tobytes() == out["tp_" + k].tobytes(), k
    # the same linear maximum as programme_loudness's dBTP (finite clips, exact mode)
    ld = b.programme_loudness(x, lengths, nchan=per, block=1000)
    live = lengths > 0
    assert np.all(np.abs(out["tp_max_dbtp"][live] - ld["tp_max"][live]) <= 1e-4)


def test_programme_truepeak_argument_errors():
    b = B()
    x = np.zeros((4, 100), np.float32)
    for kw in (dict(flags=0), dict(flags=4), dict(nchan=0), dict(block=0)):
        with pytest.raises(b.B200MError):
            b.programme_truepeak(x, [100, 100], **kw)
    with pytest.raises(b.B200MError):
        b.programme_truepeak(x, [], nchan=2)
    with pytest.raises(b.B200MError):
        b.programme_truepeak(x, [100, -1], nchan=2)
    out = b.programme_truepeak(x, [100, 50], flags=b.TPK_KMETER)
    assert "tp_hist" not in out and out["km_hist"].shape == (2, 2, 242)
