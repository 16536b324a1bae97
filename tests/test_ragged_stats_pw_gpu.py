"""GPU: ragged blocks of the bit-meter, SigDistHist and phasewheel banks (b200m_bim_run_ragged_*, b200m_sdh_run_ragged_*,
b200m_pw_process_ragged_*) and programme_stats.

Every instance is compared after every block with a private instance fed only its own frames: the first len[i] frames of each
block with len[i] > 0.  Frames at or after len[i] hold NaN, +-Inf, a denormal or 1e30 -- the values these meters count.
- bit-meter / SigDistHist: a reference plugin instance (_oracle) per bank instance, bit for bit; the bit-meter's closed flags and
  published snapshots against a private GPU bank of one run on plain blocks of that instance's lengths.
- phasewheel: a private GPU bank of one per instance, bit for bit (phase, level, peak, raw spectra); a few instances against the CPU
  port within the FFT tolerance of test_pw_gpu.py; an attached correlation bank against private reference Stcorrdsp instances.
"""
import numpy as np
import pytest

import _oracle as O
from test_stats_batch_gpu import _RefBim, _published, _script
from test_stats_gpu import _input

pytestmark = pytest.mark.gpu
FILL = (np.nan, np.inf, -np.inf, np.float32(1e-40), 1e30)
POOL = (0, 1, 31, 32, 33)
SIZES = (1024, 4097, 8192, 1024, 333, 4097, 64, 8192, 1000, 1024, 49, 4097, 1024, 1024, 2048, 1024)


def _lengths(rng, n, nfram, b, sit_out):
    """lengths 0, 1, 31, 32, 33, nfram - 1, nfram and random ones, new every block; the instances in sit_out get 0 for blocks 3..6"""
    pool = np.array([p for p in POOL if p <= nfram] + [nfram - 1, nfram, nfram])
    ln = np.where(rng.random(n) < 0.6, rng.choice(pool, n), rng.integers(0, nfram + 1, n))
    if 3 <= b <= 6:
        ln[sit_out] = 0
    if (ln == nfram).all():
        ln[0] = nfram - 1
    return ln.astype(np.int64)


def _block(x, pos, nfram, ln, per, k):
    """the block's rows, the frames at or after each instance's length overwritten with a value these meters count"""
    blk = np.array(x[:, pos:pos + nfram])
    for u, L in enumerate(ln):
        blk[u * per:(u + 1) * per, L:] = FILL[(k + u) % len(FILL)]
    return blk


def _feed(blk, host):
    import torch
    return blk if host else torch.from_numpy(blk).cuda()


def _u(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint64) if a.dtype == np.float64 else a


# ------------------------------------------------------------------------------------------------------------ bit-meter
@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("rate", [48000.0, 44100.0])
def test_bitmeter_ragged_bit_exact(rate, host):
    import meters_lv2_b200 as B
    n = 37
    cmds = [B.CTL_START, B.CTL_PAUSE, B.CTL_RESET, B.CTL_AVERAGE, B.CTL_WINDOWED, B.CTL_CLEAR]
    sc = _script(n, cmds, len(SIZES), 51)
    x = _input(n, sum(SIZES), 36)
    rng = np.random.default_rng(int(rate) + host)
    g = B.Bitmeter(n, rate)
    refs = [_RefBim(rate) for _ in range(n)]
    privs = [B.Bitmeter(1, rate) for _ in range(n)]
    pos, closes, skipped_closed = 0, 0, 0
    for b, nfram in enumerate(SIZES):
        for i in range(n):
            for c in sc[i].get(b, []):
                g.control(c, inst=i); privs[i].control(c); refs[i].cmd(c, B)
        ln = _lengths(rng, n, nfram, b, sit_out=[2, 17, 33])
        blk = _block(x, pos, nfram, ln, 1, b)
        g.run(_feed(blk, host), lengths=ln)
        assert B.lib().b200m_bim_window_closed(g.h) == 0
        for i, L in enumerate(ln):
            if L:
                row = np.ascontiguousarray(blk[i:i + 1, :L])
                refs[i].process(row)
                privs[i].run(_feed(row, host))
        pos += nfram
        r = g.results_all()
        for i, L in enumerate(ln):
            oh, oc, om, ot = refs[i].o.read(0)
            assert np.array_equal(r["hist"][i], oh), (b, i, int((r["hist"][i] != oh).sum()))
            assert np.array_equal(r["cnt"][i], oc) and np.array_equal(_u(r["minmax"][i]), _u(om)) and r["itime"][i] == ot, \
                (b, i, r["cnt"][i], oc, r["minmax"][i], om, r["itime"][i], ot)
            closed = B.lib().b200m_bim_window_closed(privs[i].h) if L else 0
            assert r["closed"][i] == closed, (b, i, L)
            closes += closed
            skipped_closed += L == 0
            ph, pc, pm, pt = _published(privs[i])
            assert np.array_equal(r["pub_hist"][i], ph) and np.array_equal(r["pub_cnt"][i], pc), (b, i)
            assert np.array_equal(_u(r["pub_minmax"][i]), _u(pm)) and r["pub_itime"][i] == pt, (b, i)
    assert closes > n // 2 and skipped_closed > n


# ------------------------------------------------------------------------------------------------------------ SigDistHist
@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("rate", [48000.0, 44100.0])
def test_sigdist_ragged_bit_exact(rate, host):
    import meters_lv2_b200 as B
    n = 35
    cmds = [B.CTL_START, B.CTL_PAUSE, B.CTL_RESET, B.CTL_CLEAR]
    sc = _script(n, cmds, len(SIZES), 52)
    for i in range(n):
        sc[i].setdefault(0, []).insert(0, B.CTL_START)                    # SigDistHist instances start paused
    x = _input(n, sum(SIZES), 37)
    rng = np.random.default_rng(int(rate) + 7 + host)
    g = B.SigDistHist(n, rate)
    refs, integ = [O.SigDist(1, rate) for _ in range(n)], [False] * n
    pos = 0
    for b, nfram in enumerate(SIZES):
        for i in range(n):
            for c in sc[i].get(b, []):
                g.control(c, inst=i)
                if c in (B.CTL_START, B.CTL_PAUSE):
                    integ[i] = c == B.CTL_START
                else:                                                      # RESET: sdh_reset; CLEAR: a new instance
                    refs[i] = O.SigDist(1, rate)
                    integ[i] = integ[i] and c == B.CTL_RESET
                refs[i].integrate(integ[i])
        ln = _lengths(rng, n, nfram, b, sit_out=[0, 9, 31])
        blk = _block(x, pos, nfram, ln, 1, b)
        g.run(_feed(blk, host), lengths=ln)
        for i, L in enumerate(ln):
            if L:
                refs[i].process(np.ascontiguousarray(blk[i:i + 1, :L]))
        pos += nfram
        h, mp, av, it = g.results_all()
        for i in range(n):
            oh, op, oa, ot = refs[i].read(0)
            assert np.array_equal(h[i], oh) and np.array_equal(mp[i], op) and it[i] == ot, (b, i, it[i], ot)
            assert np.array_equal(_u(av[i]), _u(oa)), (b, i, av[i], oa)
    assert (it > 0).sum() >= n // 3


# ------------------------------------------------------------------------------------------------------------ phasewheel
PW_SIZES = (1024, 333, 8192, 64, 4097, 1024, 8192, 49, 2000, 1024, 6000, 512)


def _pw_check(tag, g, privs, fired, pf):
    assert fired == int(any(pf)), (tag, fired, pf)
    ph, lv, pk = g.read()
    for i, p in enumerate(privs):
        oph, olv, opk = p.read()
        assert np.array_equal(_u(ph[i]), _u(oph[0])) and np.array_equal(_u(lv[i]), _u(olv[0])), (tag, i)
        assert _u(pk[i]) == _u(opk[0]), (tag, i)
        for a, c in zip(g.raw(i), p.raw(0)):
            assert np.array_equal(_u(a), _u(c)), (tag, i)


def _port_check(tag, g, o, inst):
    """raw power of instance inst against the CPU port, with test_pw_gpu.py's tolerance"""
    for a, b in zip(g.raw(inst)[:2], o.raw(0)[:2]):
        scale = b.max()
        tol = 2 * 2e-6 * np.sqrt(np.maximum(b, 0) * scale) + 1e-11 * scale
        assert (np.abs(a - b) <= tol + 1e-30).all(), (tag, inst, float(np.abs(a - b).max() / max(scale, 1e-30)))


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("bins", [64, 1024, 6144, 8192])
@pytest.mark.parametrize("mode", [0, 1])
def test_phasewheel_ragged_bit_exact(mode, bins, host):
    import meters_lv2_b200 as B
    n = 7
    rng = np.random.default_rng(1000 + bins + 10 * mode + host)
    x = (rng.uniform(-1, 1, (2 * n, sum(PW_SIZES) + 4 * 8192)) * rng.uniform(0.05, 0.9, (2 * n, 1))).astype(np.float32)
    g = B.Phasewheel(n, bins)
    privs = [B.Phasewheel(1, bins) for _ in range(n)]
    port = [O.Phasewheel(1, bins, kind="port") for _ in range(2)]
    for p in [g] + privs:
        p.set_mode(mode); p.debug_capture(True)
    for o in port:
        o.set_mode(mode)
    pos, nfired = 0, 0
    for b, nfram in enumerate(PW_SIZES):
        ln = _lengths(rng, n, nfram, b, sit_out=[1, 5])
        blk = _block(x, pos, nfram, ln, 2, b)
        fired = g.process(_feed(blk, host), lengths=ln)
        pf = []
        for i, L in enumerate(ln):
            if L:
                row = np.ascontiguousarray(blk[2 * i:2 * i + 2, :L])
                pf.append(privs[i].process(_feed(row, host)))
                if i < len(port) and port[i].process(row):
                    _port_check((mode, bins, b), g, port[i], i)
        _pw_check((mode, bins, host, b), g, privs, fired, pf)
        nfired += fired
        pos += nfram
    # plain blocks after the clocks have diverged run the per-instance form
    for nfram in (1024, 8192, 777):
        blk = np.ascontiguousarray(x[:, pos:pos + nfram])
        fired = g.process(_feed(blk, host))
        pf = [p.process(_feed(np.ascontiguousarray(blk[2 * i:2 * i + 2]), host)) for i, p in enumerate(privs)]
        _pw_check((mode, bins, host, "plain", nfram), g, privs, fired, pf)
        pos += nfram
    assert nfired >= 4


def test_phasewheel_ragged_with_attached_correlation():
    """ragged calls run the attached correlation bank over the same lengths: its readings equal private reference Stcorrdsp
    instances fed only their own frames, and the spectra still equal private phasewheel banks"""
    import meters_lv2_b200 as B
    n = 40
    rng = np.random.default_rng(77)
    x = (rng.uniform(-1, 1, (2 * n, sum(SIZES))) * rng.uniform(0.05, 0.9, (2 * n, 1))).astype(np.float32)
    g = B.Phasewheel(n, 128); cor = B.Stcorrdsp(n); g.attach_cor(cor)
    privs = [B.Phasewheel(1, 128) for _ in range(n)]
    refs = [O.Stcorr(1) for _ in range(n)]
    want = np.zeros(n, np.float32)
    for p in [g] + privs:
        p.debug_capture(True)
    pos = 0
    for b, nfram in enumerate(SIZES):
        ln = _lengths(rng, n, nfram, b, sit_out=[3, 30])
        blk = _block(x, pos, nfram, ln, 2, b)
        host = b % 3 == 2
        fired = g.process(_feed(blk, host), lengths=ln)
        pf = []
        for i, L in enumerate(ln):
            if L:
                row = np.ascontiguousarray(blk[2 * i:2 * i + 2, :L])
                refs[i].process(row); want[i] = refs[i].read()[0]
                pf.append(privs[i].process(_feed(row, True)))
        assert np.array_equal(_u(cor.read()), _u(want)), (b, np.nonzero(_u(cor.read()) != _u(want))[0][:5])
        _pw_check(("cor", b), g, privs, fired, pf)
        pos += nfram
    with pytest.raises(B.B200MError):
        cor.process(_feed(np.zeros((2 * n, 64), np.float32), False), lengths=np.full(n, 32))


# ------------------------------------------------------------------------------------------------------------ plain-call equivalence
def _equiv(make, run_plain, run_rag, read, blocks, rows):
    """two banks fed the same blocks, one plain, one ragged with every length nfram: same bits and the same launches"""
    import meters_lv2_b200 as B
    rng = np.random.default_rng(5)
    a, b = make(), make()
    for nfram in blocks:
        blk = (rng.uniform(-1, 1, (rows, nfram))).astype(np.float32)
        c0 = B.launch_count(); ra = run_plain(a, blk); c1 = B.launch_count()
        rb = run_rag(b, blk, np.full(a.n_inst, nfram)); c2 = B.launch_count()
        assert c1 - c0 == c2 - c1 and ra == rb, (nfram, c1 - c0, c2 - c1)
        for u, v in zip(read(a), read(b)):
            assert np.array_equal(_u(u), _u(v)), nfram


def test_all_nfram_ragged_calls_are_plain_calls():
    import torch
    import meters_lv2_b200 as B
    dev = lambda blk: torch.from_numpy(blk).cuda()                       # noqa: E731
    blocks = (1024, 64, 8192, 1000, 1024)

    def bim():
        g = B.Bitmeter(20); g.control(B.CTL_AVERAGE); return g
    bim_read = lambda g: [g.results_all()[k] for k in ("hist", "cnt", "minmax", "itime", "closed", "pub_hist")] + \
        [np.int32(B.lib().b200m_bim_window_closed(g.h))]                  # noqa: E731
    _equiv(bim, lambda g, x: g.run(dev(x)), lambda g, x, ln: g.run(dev(x), lengths=ln), bim_read, blocks, 20)

    def sdh():
        g = B.SigDistHist(20); g.control(B.CTL_START); return g
    _equiv(sdh, lambda g, x: g.run(x), lambda g, x, ln: g.run(x, lengths=ln), lambda g: g.results_all(), blocks, 20)

    def pw(attach):
        def make():
            g = B.Phasewheel(6, 256)
            if attach:
                g._c = B.Stcorrdsp(6); g.attach_cor(g._c)
            return g
        return make
    pw_read = lambda g: list(g.read()) + ([g._c.read()] if hasattr(g, "_c") else [])   # noqa: E731
    for attach in (False, True):
        _equiv(pw(attach), lambda g, x: g.process(dev(x)), lambda g, x, ln: g.process(dev(x), lengths=ln), pw_read, blocks, 12)


# ------------------------------------------------------------------------------------------------------------ refusals
def test_ragged_refusals_leave_the_banks_alone():
    import torch
    import meters_lv2_b200 as B
    n = 10
    x = torch.from_numpy(np.random.default_rng(3).uniform(-1, 1, (2 * n, 256)).astype(np.float32)).cuda()
    bim, sdh, pw = B.Bitmeter(n), B.SigDistHist(n), B.Phasewheel(n, 64)
    sdh.control(B.CTL_START)
    runs = [(bim, lambda ln: bim.run(x[:n], lengths=ln), lambda: bim.results_all()),
            (sdh, lambda ln: sdh.run(x[:n], lengths=ln), lambda: sdh.results_all()),
            (pw, lambda ln: pw.process(x, lengths=ln), lambda: pw.read())]
    for g, run, read in runs:
        run(np.arange(n) * 20)                                             # ragged: the phasewheel clocks diverge
        torch.cuda.synchronize()
        before = read()
        before = list(before.values()) if isinstance(before, dict) else list(before)
        for bad in (np.full(n, 257), np.full(n - 1, 5), np.full(n + 1, 5)):
            c0 = B.launch_count()
            with pytest.raises(B.B200MError):
                run(bad)
            assert B.launch_count() == c0
        after = read()
        after = list(after.values()) if isinstance(after, dict) else list(after)
        for u, v in zip(before, after):
            assert np.array_equal(_u(u), _u(v))
        run(np.full(n, 256))                                              # the bank still runs
    # the C entry points refuse a length above nfram themselves (the Python wrapper checks only the count)
    ln = np.full(n, 300, np.uint32)
    p, s, _, nf = B._dev_ptr(x[:n])
    assert B.lib().b200m_bim_run_ragged_device(bim.h, p, s, nf, B._np_ptr(ln), B._stream_ptr(None)) == -1
    assert B.lib().b200m_sdh_run_ragged_device(sdh.h, p, s, nf, B._np_ptr(ln), B._stream_ptr(None)) == -1


# ------------------------------------------------------------------------------------------------------------ programme_stats
@pytest.mark.parametrize("host", [False, True])
def test_programme_stats_equals_whole_clip_reference(host):
    import torch
    import meters_lv2_b200 as B
    lengths = np.array([0, 1, 1023, 1024, 1025, 48000, 100003, 240000, 17, 4096 * 3 + 5, 200000, 33])
    n = lengths.size
    x = _input(n, int(lengths.max()), 38)
    x[5, 100:200] = np.float32(1e-41)
    x[7, 5000] = np.nan; x[7, 6000] = -np.inf
    for i, L in enumerate(lengths):
        x[i, L:] = FILL[i % len(FILL)]
    r = B.programme_stats(x if host else torch.from_numpy(x).cuda(), lengths, block=1000 if host else 1024)
    for i, L in enumerate(lengths):
        bo = O.Bitmeter(1); bo.mode(True, True)
        so = O.SigDist(1); so.integrate(True)
        for o in range(0, L, 8192):                                        # the whole clip, in plugin-sized runs
            row = np.ascontiguousarray(x[i:i + 1, o:min(L, o + 8192)])
            bo.process(row); so.process(row)
        oh, oc, om, ot = bo.read(0)
        assert np.array_equal(r["bim_hist"][i], oh) and np.array_equal(r["bim_cnt"][i], oc), (i, L)
        assert np.array_equal(_u(r["bim_minmax"][i]), _u(om)) and r["bim_itime"][i] == ot, (i, L, r["bim_minmax"][i], om)
        sh, sp, sa, st = so.read(0)
        assert np.array_equal(r["sdh_hist"][i], sh) and np.array_equal(r["sdh_max_peak"][i], sp) and r["sdh_itime"][i] == st, (i, L)
        assert np.array_equal(_u(r["sdh_avg_tmp_var"][i]), _u(sa)), (i, L)
    assert r["bim_itime"][7] == 240000 and r["bim_cnt"][7, 2] >= 1 and r["bim_cnt"][7, 3] >= 1
