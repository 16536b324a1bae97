"""GPU: the loudness log of the EBU R128 bank (b200m_ebu_log_enable / b200m_ebu_log_drain) and programme_loudness(curves=True).

The oracle of a logged point is a private reference instance per bank instance (the reference build when present, else the port;
the restatement in tests/_ebu_weighted.cc for weighted layouts) fed the same blocks, each additionally cut at the instance's own
50 ms fragment edges, and read after every edge.  The reference cuts its process() calls at those edges itself
(ebu_r128_proc.cc:212-216), so the extra cuts change nothing; a cut anywhere else would.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _ebu_weighted as W
import _oracle as O
import _signals as S

pytestmark = pytest.mark.gpu
POINT_COLS = [0, 2, 4, 6, 7]          # loudness_M, loudness_S, integrated, range_min, range_max of an oracle read()
RES = ("loudness_M", "loudness_S", "integrated", "range_min", "range_max")


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def sig(nrows, off, nfram, seed=11):
    """frames off .. off + nfram - 1 of a seeded stream whose level swings over some 50 dB, at another rate on every instance"""
    x = S.white(nrows, nfram, seed=seed, block=off)
    t = (off + np.arange(nfram, dtype=np.float64)) / 48000.0
    per = 2.0 + (np.arange(nrows) // 2 % 7)[:, None]
    env = 10.0 ** ((-28.0 + 25.0 * np.sin(2 * np.pi * t[None, :] / per)) / 20.0)
    return np.ascontiguousarray(x * env, np.float32)


class _Oracle:
    """one private reference instance per bank instance, each process() cut at its own fragment edges, a point after each edge"""

    def __init__(self, n, fs=48000.0, nchan=2, gains=None):
        self.nc = nchan if gains is None else len(gains)
        self.e = [O.Ebu(1, nchan, fs) if gains is None else W.Ebu(1, gains, fs) for _ in range(n)]
        self.fragm = int(fs) // 20
        self.left = [self.fragm] * n
        self.pts = [[] for _ in range(n)]

    def integr(self, cmd, inst=-1):
        for i in (range(len(self.e)) if inst < 0 else [inst]):
            self.e[i].integr(cmd)

    def reset(self, i):
        self.e[i].reset()
        self.left[i] = self.fragm

    def process(self, x, lens=None, only=None):
        for i in (range(len(self.e)) if only is None else only):
            L = x.shape[1] if lens is None else int(lens[i])
            a = 0
            while a < L:
                k = min(self.left[i], L - a)
                self.e[i].process(np.ascontiguousarray(x[i * self.nc:(i + 1) * self.nc, a:a + k]))
                a += k
                self.left[i] -= k
                if self.left[i] == 0:
                    self.pts[i].append(self.e[i].read()[0, POINT_COLS])
                    self.left[i] = self.fragm

    def points(self, i):
        return np.asarray(self.pts[i], np.float32).reshape(-1, 5)


class _Acc:
    """the drained points of every instance, concatenated over drains"""

    def __init__(self, n):
        self.p = [[] for _ in range(n)]

    def drain(self, bank, stream=None):
        pts, cnt, lost = bank.log_drain(stream)
        assert not lost.any()
        f = pts.view(np.float32).reshape(pts.shape[0], pts.shape[1], 5)
        for i in range(len(self.p)):
            self.p[i].append(f[i, :cnt[i]])
        return cnt

    def points(self, i):
        return np.concatenate(self.p[i]).reshape(-1, 5)


def _same(acc, orc, insts):
    for i in insts:
        a, b = acc.points(i), orc.points(i)
        assert a.shape == b.shape, (i, a.shape, b.shape)
        assert np.array_equal(u32(a), u32(b)), "instance %d: first differing point %s" % (i, np.argwhere(u32(a) != u32(b))[:1])


# ---- 1. oracle parity with controls mid-run ---------------------------------------------------------------------------------
@pytest.mark.parametrize("fs,block", [(48000.0, 1024), (48000.0, 8192), (44100.0, 1024)])
def test_log_matches_oracle_with_controls(fs, block):
    import meters_lv2_b200 as B
    n = 64
    nb = -(-int(30 * fs) // block)
    bank = B.Ebu_r128_proc(n, 2, fs)
    bank.log_enable(1024)
    orc = _Oracle(n, fs)
    acc = _Acc(n)
    bank.integr_start(); orc.integr("start")
    for b in range(nb):
        if b == nb // 4:
            bank.integr_pause(); orc.integr("pause")
        if b == 3 * nb // 8:
            bank.integr_start(); orc.integr("start")
        if b == nb // 2:
            for i in range(0, n, 5):                       # their clocks restart here: several fragment phases from now on
                bank.reset(i); orc.reset(i)
            acc.drain(bank)
        if b == 5 * nb // 8:
            bank.integr_start(); orc.integr("start")
        x = sig(2 * n, b * block, block)
        bank.process(torch.from_numpy(x).cuda())
        orc.process(x)
    acc.drain(bank)
    _same(acc, orc, range(n))
    res = bank.results()
    for i in range(n):                                     # the last point is what results() reads
        last = acc.points(i)[-1]
        assert all(u32(last[k]) == u32(res[f][i]) for k, f in enumerate(RES)), i


# ---- 2. ragged blocks and programme_loudness(curves=True) -------------------------------------------------------------------
@pytest.mark.parametrize("block", [1024, 8192])
def test_programme_loudness_curves(block):
    import meters_lv2_b200 as B
    fs, fragm = 48000.0, 2400
    lengths = np.array([0, 1000, 7 * fragm, 3 * 60 * 48000 + 777, 50 * fragm + 123, fragm, 95 * fragm], np.int64)
    n = lengths.size
    get = lambda off, m: sig(2 * n, off, m, seed=5)
    out = B.programme_loudness(get, lengths, fs, block=block, curves=True)
    ref = B.programme_loudness(get, lengths, fs, block=block)
    for k, v in ref.items():
        assert np.array_equal(np.asarray(out[k]).view(np.uint32), np.asarray(v).view(np.uint32)), k
    assert out["n_points"].dtype == np.int64 and np.array_equal(out["n_points"], lengths // fragm)
    width = int((lengths // fragm).max())
    orc = _Oracle(n, fs)
    orc.integr("start")
    total = int(lengths.max())
    for off in range(0, total, block):
        m = min(block, total - off)
        orc.process(get(off, m), lens=np.clip(lengths - off, 0, m))
    for k, f in enumerate(("curve_M", "curve_S", "curve_I", "curve_range_min", "curve_range_max")):
        c = out[f]
        assert c.dtype == np.float32 and c.shape == (n, width), f
        for i in range(n):
            npt = int(lengths[i] // fragm)
            assert np.array_equal(u32(c[i, :npt]), u32(orc.points(i)[:, k])), (f, i)
            assert np.isnan(c[i, npt:]).all(), (f, i)


def test_ragged_log_matches_oracle():
    import meters_lv2_b200 as B
    n, nf, fs = 48, 1024, 48000.0
    rng = np.random.default_rng(3)
    bank = B.Ebu_r128_proc(n, 2, fs)
    bank.log_enable(256)
    orc = _Oracle(n, fs)
    acc = _Acc(n)
    bank.integr_start(); orc.integr("start")
    for b in range(400):
        lens = np.full(n, nf, np.uint32)
        if b % 3 == 1:
            k = rng.choice(n, n // 3, replace=False)
            lens[k] = rng.integers(0, nf, k.size)
        x = sig(2 * n, b * nf, nf, seed=9)
        x[np.arange(nf)[None, :] >= np.repeat(lens, 2)[:, None]] = np.nan      # frames past an instance's length are never read
        bank.process(torch.from_numpy(x).cuda(), lengths=lens)
        orc.process(x, lens=lens)
        if b % 150 == 149:
            acc.drain(bank)
    acc.drain(bank)
    _same(acc, orc, range(n))


# ---- 3. every path gives the same log ---------------------------------------------------------------------------------------
def _drive(bank, n, nblocks, nf, dev, ragged=True, seed=21, run="process"):
    """the same schedule on any bank: integration on, a reset of every 4th instance mid-run, a ragged block; the drained points"""
    acc = _Acc(n)
    is_r128 = run == "run"
    if is_r128:
        bank.control(bank.START)
    else:
        bank.integr_start()
    for b in range(nblocks):
        if b == nblocks // 2:
            for i in range(0, n, 4):
                if is_r128:
                    bank.control(bank.NEW, i); bank.control(bank.START, i)
                else:
                    bank.reset(i); bank.integr_start(i)
        x = sig(bank.nchan * n, b * nf, nf, seed=seed)
        xin = torch.from_numpy(x).cuda() if dev else x
        lens = None
        if ragged and b == nblocks // 3:
            lens = np.full(n, nf, np.uint32); lens[1::3] = nf // 3
        getattr(bank, run)(xin, lengths=lens)
        if b == nblocks - 40:
            acc.drain(bank)
    acc.drain(bank)
    return acc


def _same_acc_n(a, b, n, npts):
    for i in range(n):
        assert a.points(i).shape[0] == npts and np.array_equal(u32(a.points(i)), u32(b.points(i))), i


def _same_acc(a, b, n):
    for i in range(n):
        assert np.array_equal(u32(a.points(i)), u32(b.points(i))), i
        assert a.points(i).shape[0] > 50


def test_device_and_host_paths_log_the_same():
    import meters_lv2_b200 as B
    n = 96
    for make, run in ((lambda: B.Ebu_r128_proc(n, 2), "process"), (lambda: B.EBUr128(n, 48000.0, True), "run")):
        logs = []
        for dev in (True, False):                          # EBUr128.run on numpy: the sliced host path
            bank = make(); bank.log_enable(512)
            logs.append(_drive(bank, n, 200, 1024, dev, run=run))
            bank.close()
        _same_acc(logs[0], logs[1], n)


def test_host_path_drain_is_ordered_after_the_cycle():
    """an EBUr128 bank on the host path runs its kernels on its own (non-blocking) stream: a drain right behind run(), with no
    results() in between, must still see every point of the last block, gated"""
    import meters_lv2_b200 as B
    n, nf, nb = 4096, 1024, 50
    logs, cnts = [], []
    for dev in (True, False):
        bank = B.EBUr128(n, 48000.0, True); bank.set_precision(B.PREC_EXACT); bank.log_enable(64)
        bank.control(bank.START)
        acc = _Acc(n)
        for b in range(nb):
            x = sig(2 * n, b * nf, nf, seed=8)
            bank.run(torch.from_numpy(x).cuda() if dev else x)
            if b in (23, nb - 1):                          # fragments end in blocks 23 (frame 24000) and 49 (frame 50400)
                cnts.append(acc.drain(bank).copy())
        logs.append(acc)
        bank.close()
    assert all((c == k).all() for c, k in zip(cnts, (10, 11, 10, 11))), [np.unique(c) for c in cnts]
    _same_acc_n(logs[0], logs[1], n, 21)


def test_tma_k1_logs_the_same(monkeypatch):
    import meters_lv2_b200 as B
    n = 64
    logs = []
    for tma in ("0", "1"):
        monkeypatch.setenv("B200M_EBU_TMA", tma)           # read when the bank is created
        bank = B.Ebu_r128_proc(n, 2); bank.log_enable(256)
        logs.append(_drive(bank, n, 150, 1024, True, ragged=False))
        bank.close()
    _same_acc(logs[0], logs[1], n)


def test_fused_tolerance_bank_logs_like_exact():
    import meters_lv2_b200 as B
    n = 5120                                               # 10240 channels: the fused K-weighting + true-peak kernel
    banks = []
    for prec in (B.PREC_FMA, B.PREC_EXACT):
        bank = B.EBUr128(n, 48000.0, True); bank.set_precision(prec); bank.log_enable(128)
        bank.control(bank.START)
        banks.append(bank)
    base = torch.from_numpy(sig(2 * n, 0, 4096, seed=4)).cuda()
    for b in range(120):
        s = (b * 1024) % 3072
        x = base[:, s:s + 1024] * (0.25 + 0.75 * ((b // 7) % 4) / 3)
        d = []
        for bank in banks:
            l0 = B.launch_count(); bank.run(x); d.append(B.launch_count() - l0)
        assert d[1] - d[0] == 1, (b, d)                    # the fused kernel ran in place of K1 + the true-peak kernel
    logs = [_Acc(n), _Acc(n)]
    for acc, bank in zip(logs, banks):
        acc.drain(bank)
    _same_acc(logs[0], logs[1], n)


@pytest.mark.parametrize("layout", ["7.1.4+lfe", "5ch", "mono"])
def test_weighted_surround_mono_logs_match_oracle(layout):
    import meters_lv2_b200 as B
    fs, nf = 48000.0, 1024
    if layout == "7.1.4+lfe":
        g = np.concatenate([B.bs1770_weights([30, -30, 0, 90, -90, 135, -135, 45, -45, 135, -135], [0] * 7 + [35] * 4), [0.0]])
        n, nchan, bank = 40, 12, B.Ebu_r128_proc(40, 12, fs, gains=g.astype(np.float32))
    else:
        g = None
        nchan = 5 if layout == "5ch" else 1
        n = 70
        bank = B.Ebu_r128_proc(n, nchan, fs)
    sub = [0, 1, 17, n - 1]
    bank.log_enable(256)
    orc = _Oracle(n, fs, nchan, gains=None if g is None else g.astype(np.float32))
    acc = _Acc(n)
    bank.integr_start(); orc.integr("start")
    for b in range(300):
        if b == 120:
            bank.reset(17); orc.reset(17); bank.integr_start(17); orc.integr("start", 17)
        x = sig(nchan * n, b * nf, nf, seed=2)
        bank.process(torch.from_numpy(x).cuda())
        orc.process(x, only=sub)
    acc.drain(bank)
    _same(acc, orc, sub)


# ---- 4. consistency at scale ------------------------------------------------------------------------------------------------
def test_scale_8192_consistency():
    import meters_lv2_b200 as B
    n, nf, nb = 8192, 1024, 470
    bank = B.EBUr128(n, 48000.0, True)
    bank.log_enable(256)
    bank.control(bank.START)
    g = torch.Generator(device="cuda").manual_seed(1)
    base = torch.rand(2 * n, 4 * nf, device="cuda", generator=g) * 2 - 1
    lvl = torch.rand(n, 16, device="cuda", generator=g).repeat_interleave(2, 0) ** 3
    for b in range(nb):
        s = (b % 4) * nf
        bank.run(base[:, s:s + nf] * lvl[:, (b // 9) % 16, None])
    pts, cnt, lost = bank.log_drain()
    res, _ = bank.results()
    assert (cnt == nb * nf // 2400).all() and not lost.any()
    last = pts[np.arange(n), cnt.astype(np.int64) - 1]
    for f in RES:
        assert np.array_equal(u32(last[f]), u32(res[f])), f
    assert np.array_equal(u32(np.nanmax(pts["loudness_M"], axis=1)), u32(res["maxloudn_M"]))
    assert np.array_equal(u32(np.nanmax(pts["loudness_S"], axis=1)), u32(res["maxloudn_S"]))


# ---- 5. ring semantics ------------------------------------------------------------------------------------------------------
def test_ring_keeps_the_last_capacity_points():
    import meters_lv2_b200 as B
    n, cap = 37, 7
    small, big = B.Ebu_r128_proc(n, 2), B.Ebu_r128_proc(n, 2)
    small.log_enable(cap); big.log_enable(64)
    for bank in (small, big):
        bank.integr_start()
    for b in range(50):                                    # 50 x 1024 frames: 21 fragments
        x = torch.from_numpy(sig(2 * n, b * 1024, 1024)).cuda()
        small.process(x); big.process(x)
    p, c, lost = small.log_drain()
    q, d, _ = big.log_drain()
    assert (d == 21).all() and (c == cap).all() and (lost == 21 - cap).all()
    assert np.array_equal(u32(p.view(np.float32)), u32(np.ascontiguousarray(q[:, 21 - cap:21]).view(np.float32)))
    p, c, lost = small.log_drain()
    assert not c.any() and not lost.any() and np.isnan(p.view(np.float32)).all()
    for b in range(50, 53):                                # frames 51200 .. 54271: the fragment ending at 52800
        small.process(torch.from_numpy(sig(2 * n, b * 1024, 1024)).cuda())
    small.log_enable(cap)                                  # re-enabling empties the log
    assert not small.log_drain()[1].any()
    small.process(torch.from_numpy(sig(2 * n, 53 * 1024, 1024)).cuda())    # ... and it logs on: the fragment ending at 55200
    assert (small.log_drain()[1] == 1).all()


# ---- 6. no behaviour change -------------------------------------------------------------------------------------------------
def test_log_changes_nothing_else():
    import meters_lv2_b200 as B
    n = 96
    on, off = B.EBUr128(n, 48000.0, True), B.EBUr128(n, 48000.0, True)
    on.log_enable(300)
    assert B.lib().b200m_r128_snapshot_size(on.h) == B.lib().b200m_r128_snapshot_size(off.h)
    for bank in (on, off):
        bank.control(bank.START)
    for b in range(260):
        x = torch.from_numpy(sig(2 * n, b * 2048, 2048)).cuda()
        if b == 100:
            for bank in (on, off):
                bank.control(bank.NEW, 3); bank.control(bank.START, 3); bank.control(bank.PAUSE, 9)
        d = []
        for bank in (on, off):
            torch.cuda.synchronize()
            l0 = B.launch_count()
            bank.run(x)
            d.append(B.launch_count() - l0)
        assert d[0] == d[1], b
    (ra, ta), (rb, tb) = on.results(), off.results()
    assert ra.tobytes() == rb.tobytes() and ta.tobytes() == tb.tobytes()
    for i in (0, 3, 9, n - 1):
        assert all(np.array_equal(u, v) for u, v in zip(on.histogram(i), off.histogram(i)))
    assert on.snapshot().tobytes() == off.snapshot().tobytes()
    # a snapshot restored into a bank whose log is on: it keeps logging, like the bank it was taken from
    snap = off.snapshot()
    on.log_drain()
    other = B.EBUr128(n, 48000.0, True)
    other.log_enable(300)
    other.restore(snap)
    accs = [_Acc(n), _Acc(n)]
    for b in range(80):
        x = torch.from_numpy(sig(2 * n, (260 + b) * 2048, 2048)).cuda()
        on.run(x); other.run(x)
    for acc, bank in zip(accs, (on, other)):
        acc.drain(bank)
    _same_acc(accs[0], accs[1], n)


# ---- 7. streams and errors --------------------------------------------------------------------------------------------------
def test_drain_on_caller_stream_sees_every_point():
    import meters_lv2_b200 as B
    n = 512
    bank = B.EBUr128(n, 48000.0, True)
    s = torch.cuda.Stream()
    bank.log_enable(256, stream=s)
    bank.control(bank.START, stream=s)
    xs = torch.from_numpy(sig(2 * n, 0, 8192)).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for b in range(60):
            bank.run(xs, stream=s)
        pts, cnt, lost = bank.log_drain(stream=s)          # no synchronisation in between
    assert (cnt == 60 * 8192 // 2400).all() and not lost.any()
    assert not np.isnan(pts.view(np.float32).reshape(n, -1, 5)[:, :int(cnt[0])]).any()


def test_log_errors_are_codes():
    import meters_lv2_b200 as B
    L = B.lib()
    bank = B.Ebu_r128_proc(1024, 2)
    with pytest.raises(B.B200MError, match="log is off"):
        bank.log_drain()
    pts = np.empty((1024, 4), B.EBU_POINT_DTYPE); cnt = np.empty(1024, np.uint32); lost = np.empty(1024, np.uint64)
    assert L.b200m_ebu_log_drain(bank.h, B._np_ptr(pts), B._np_ptr(cnt), B._np_ptr(lost), None) == -1
    assert L.b200m_ebu_log_enable(None, 4, None) == -1
    assert L.b200m_ebu_log_capacity(bank.h) == 0 and L.b200m_ebu_log_capacity(None) == 0
    bank.log_enable(4)
    assert L.b200m_ebu_log_capacity(bank.h) == 4
    L.b200m_ebu_log_enable(bank.h, 9, None)                # enabled behind the wrapper's back: the drain sizes its buffer from the bank
    assert bank.log_drain()[0].shape == (1024, 9)
    bank.log_enable(4)
    assert L.b200m_ebu_log_drain(None, B._np_ptr(pts), B._np_ptr(cnt), B._np_ptr(lost), None) == -1
    assert L.b200m_ebu_log_drain(bank.h, None, B._np_ptr(cnt), B._np_ptr(lost), None) == -1
    assert L.b200m_ebu_log_drain(bank.h, B._np_ptr(pts), None, B._np_ptr(lost), None) == -1
    assert L.b200m_ebu_log_drain(bank.h, B._np_ptr(pts), B._np_ptr(cnt), None, None) == -1
    # a capacity no device can hold: B200M_E_NOMEM, the log is off, and the bank keeps working
    assert L.b200m_ebu_log_enable(bank.h, C.c_uint32(0xFFFFFFFF), None) == -2
    with pytest.raises(B.B200MError, match="log is off"):
        bank.log_drain()
    bank.integr_start()
    for b in range(3):
        bank.process(torch.from_numpy(sig(2048, b * 2400, 2400)).cuda())
    assert (bank.results()["frag_power"] > 0).all()
    bank.log_enable(0)
    with pytest.raises(B.B200MError):
        bank.log_drain()
