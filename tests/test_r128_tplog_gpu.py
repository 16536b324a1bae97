"""GPU: true-peak curves, the dBTP plane of the EBUr128 bank's loudness log (b200m_r128_log_enable / b200m_r128_log_drain) and
programme_loudness(curves=True)'s curve_TP.

The oracle of a point's dBTP is a second private TruePeakdsp per channel of each bank instance (the reference build when present,
else the port).  It gets exactly the process_max calls the plugin's own meters get (none while the instance's dBTP is off; a
ragged block's first len[i] frames), each also cut at the instance's 50 ms fragment edges.  process_max starts its maximum afresh
after a read() (truepeakdsp.cc:110) and never clears the read latch, so the oracle reads after every call and keeps the largest
read of the fragment over the instance's channels; at each edge the point is coef_to_db of that, 0 (-inf dBTP) when the fragment
ran nothing.  The 4x FIR is causal and its output does not depend on where process_max calls are cut, so the extra cuts change no
output.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _oracle as O
import _signals as S

pytestmark = pytest.mark.gpu
_libm = C.CDLL("libm.so.6")
_libm.log10f.restype = C.c_float
_libm.log10f.argtypes = [C.c_float]


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _db(v):
    """coef_to_db (src/ebulv2.cc:227-230): 20.0 * log10f (val), the double product rounded to float"""
    return np.float32(-np.inf) if v == 0 else np.float32(20.0 * float(_libm.log10f(float(v))))


def sig(nrows, off, nfram, seed=11, fs=48000.0):
    """frames off .. off + nfram - 1 of a seeded stream whose level swings over some 50 dB, at another rate on every instance"""
    x = S.white(nrows, nfram, seed=seed, block=off)
    t = (off + np.arange(nfram, dtype=np.float64)) / fs
    per = 2.0 + (np.arange(nrows) // 2 % 7)[:, None]
    env = 10.0 ** ((-28.0 + 25.0 * np.sin(2 * np.pi * t[None, :] / per)) / 20.0)
    return np.ascontiguousarray(x * env, np.float32)


class _TpOracle:
    """per bank instance a private TruePeakdsp set, each process_max cut at the instance's fragment edges, read after each edge"""

    def __init__(self, n, nc, fs=48000.0):
        self.n, self.nc, self.fs = n, nc, fs
        self.fragm = int(fs) // 20
        self.tp = [O.TruePeak(nc, fs) for _ in range(n)]
        self.left = [self.fragm] * n
        self.mx = [np.float32(0)] * n                     # the largest read of the open fragment
        self.on = [True] * n
        self.pts = [[] for _ in range(n)]

    def new(self, i):
        """B200M_R128_NEW: fresh meters, the fragment clock restarts with the next block"""
        self.clear(i)
        self.left[i] = self.fragm

    def clear(self, i):
        """B200M_R128_CLEAR: fresh meters, the clock runs on; the open fragment's frames so far no longer count"""
        self.tp[i] = O.TruePeak(self.nc, self.fs)
        self.mx[i] = np.float32(0)

    def cut(self, i):
        """the open fragment's frames so far no longer count (a restore), the meters' histories stay"""
        self.mx[i] = np.float32(0)

    def process(self, x, lens=None, only=None):
        for i in (range(self.n) if only is None else only):
            L = x.shape[1] if lens is None else int(lens[i])
            a = 0
            while a < L:
                k = min(self.left[i], L - a)
                if self.on[i]:
                    self.tp[i].process(np.ascontiguousarray(x[i * self.nc:(i + 1) * self.nc, a:a + k]), mode=1)
                    m, _ = self.tp[i].read()
                    for c in range(self.nc):
                        self.mx[i] = self.mx[i] if self.mx[i] > m[c] else m[c]
                a += k
                self.left[i] -= k
                if self.left[i] == 0:
                    self.pts[i].append(_db(self.mx[i]))
                    self.mx[i] = np.float32(0)
                    self.left[i] = self.fragm

    def points(self, i):
        return np.asarray(self.pts[i], np.float32)


class _Acc:
    """the drained points of every instance, concatenated over drains: [npts, 6] float32 per instance"""

    def __init__(self, n):
        self.p = [[] for _ in range(n)]

    def drain(self, bank, stream=None):
        pts, cnt, lost = bank.log_drain(stream)
        assert not lost.any()
        nf = len(pts.dtype.names)
        f = pts.view(np.float32).reshape(pts.shape[0], pts.shape[1], nf)
        assert np.isnan(f[np.arange(pts.shape[1])[None, :] >= cnt[:, None].astype(np.int64)]).all()
        for i in range(len(self.p)):
            self.p[i].append(f[i, :cnt[i]])
        return cnt

    def points(self, i):
        return np.concatenate(self.p[i])


def _same_tp(acc, orc, insts, tag=""):
    for i in insts:
        a, b = acc.points(i)[:, 5], orc.points(i)
        assert a.shape == b.shape, (tag, i, a.shape, b.shape)
        bad = np.nonzero(u32(a) != u32(b))[0]
        assert bad.size == 0, "%s instance %d: point %d is %r, oracle %r" % (tag, i, bad[0], a[bad[0]], b[bad[0]])


def _same_all(a, b, n, nfields=6):
    for i in range(n):
        assert np.array_equal(u32(a.points(i)[:, :nfields]), u32(b.points(i)[:, :nfields])), i


# ---- 1. bit-exact against the oracle in exact mode, with controls and dBTP switches mid-run --------------------------------------
@pytest.mark.parametrize("fs,block", [(48000.0, 1024), (48000.0, 8192), (44100.0, 1024), (44100.0, 8192)])
def test_points_match_oracle_with_controls(fs, block):
    import meters_lv2_b200 as B
    n = 24
    nb = -(-int(20 * fs) // block)
    plane, loud, off = (B.EBUr128(n, fs, True) for _ in range(3))
    for bank in (plane, loud, off):
        bank.set_precision(B.PREC_EXACT)
        bank.control(bank.START)
    plane.log_enable(1024, dbtp=True)
    loud.log_enable(1024)
    orc = _TpOracle(n, 2, fs)
    accs = [_Acc(n), _Acc(n)]
    banks = (plane, loud, off)
    for b in range(nb):
        if b == nb // 5:
            for bank in banks:
                bank.control(bank.PAUSE)
        if b == 3 * nb // 10:
            for bank in banks:
                bank.control(bank.START)
        if b == 2 * nb // 5:
            for i in range(0, n, 3):                       # RESET: integration and the hold restart, the open fragment runs on
                for bank in banks:
                    bank.control(bank.RESET, i)
        if b == nb // 2:
            for acc, bank in zip(accs, (plane, loud)):
                acc.drain(bank)
            for i in range(1, n, 4):                       # NEW: a fresh plugin whose clock starts with the next block
                for bank in banks:
                    bank.control(bank.NEW, i); bank.control(bank.START, i)
                orc.new(i)
            for bank in banks:                             # CLEAR: a fresh plugin on the running clock
                bank.control(bank.CLEAR, 6); bank.control(bank.START, 6)
            orc.clear(6)
        if b == 3 * nb // 5:
            for i in range(2, n, 5):
                for bank in banks:
                    bank.set_dbtp(False, i)
                orc.on[i] = False
        if b == 7 * nb // 10:                              # three blocks with no instance metering dBTP: no true-peak kernel runs
            for bank in banks:
                bank.set_dbtp(False)
            orc.on = [False] * n
        if b == 7 * nb // 10 + 3:
            for bank in banks:
                bank.set_dbtp(True)
                for i in range(2, n, 5):
                    bank.set_dbtp(False, i)
            orc.on = [i % 5 != 2 for i in range(n)]
        if b == 4 * nb // 5:
            for bank in banks:
                bank.set_dbtp(True)
            orc.on = [True] * n
        x = sig(2 * n, b * block, block, fs=fs)
        xd = torch.from_numpy(x).cuda()
        for bank in banks:
            bank.run(xd)
        orc.process(x)
    for acc, bank in zip(accs, (plane, loud)):
        acc.drain(bank)
    _same_tp(accs[0], orc, range(n))
    assert any(np.isneginf(accs[0].points(i)[:, 5]).any() for i in range(2, n, 5))
    # the five loudness fields are those of a loudness-only log, every result and the hold those of a bank without a log
    _same_all(accs[0], accs[1], n, 5)
    (ra, ta), (rb, tb), (rc, tc) = plane.results(), loud.results(), off.results()
    assert ra.tobytes() == rc.tobytes() and rb.tobytes() == rc.tobytes()
    assert u32(ta).tobytes() == u32(tc).tobytes() and u32(tb).tobytes() == u32(tc).tobytes()


# ---- 2. every path gives the same points: ragged blocks, channel counts, weighted layouts, host path --------------------------------
@pytest.mark.parametrize("layout,dev", [("stereo", False), ("stereo", True), ("mono", True), ("3ch", True), ("5ch", True),
                                        ("7.1.4+lfe", True)])
def test_paths_and_layouts_match_oracle(layout, dev):
    import meters_lv2_b200 as B
    fs, nf = 48000.0, 1024
    rng = np.random.default_rng(7)
    if layout == "7.1.4+lfe":
        g = np.concatenate([B.bs1770_weights([30, -30, 0, 90, -90, 135, -135, 45, -45, 135, -135], [0] * 7 + [35] * 4), [0.0]])
        n, nc = 16, 12
        bank = B.EBUr128(n, fs, True, nchan=nc, gains=g.astype(np.float32))
    else:
        nc = {"stereo": 2, "mono": 1, "3ch": 3, "5ch": 5}[layout]
        n = 64 if not dev else 24                          # the host path cuts banks of >= 64 instances into slices
        bank = B.EBUr128(n, fs, True, nchan=nc)
    bank.set_precision(B.PREC_EXACT)
    bank.log_enable(512, dbtp=True)
    bank.control(bank.START)
    orc = _TpOracle(n, nc, fs)
    acc = _Acc(n)
    for b in range(240):
        x = sig(nc * n, b * nf, nf, seed=3)
        if layout == "7.1.4+lfe":
            x[11::12] *= 4.0 * (b % 3)                     # the LFE row (weight 0) sets the true peak now and then
        lens = None
        if b % 3 == 1:
            lens = np.full(n, nf, np.uint32)
            k = rng.choice(n, n // 3, replace=False)
            lens[k] = rng.integers(0, nf, k.size)
            x[np.arange(nf)[None, :] >= np.repeat(lens, nc)[:, None]] = np.nan       # frames past a length are never read
        bank.run(torch.from_numpy(x).cuda() if dev else x, lengths=lens)
        orc.process(x, lens=lens)
        if b == 150:
            acc.drain(bank)
    acc.drain(bank)
    _same_tp(acc, orc, range(n), layout)


def test_host_path_drain_is_ordered_after_the_cycle():
    """the sliced host path runs the true-peak kernels on a side stream: a drain right behind run(), with nothing in between, sees
    every point of the last block, dBTP included, the same as on the device path"""
    import meters_lv2_b200 as B
    n, nf, nb = 2048, 1024, 50
    logs, cnts = [], []
    for dev in (True, False):
        bank = B.EBUr128(n, 48000.0, True); bank.set_precision(B.PREC_EXACT); bank.log_enable(64, dbtp=True)
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
    for i in range(n):
        assert logs[0].points(i).shape == (21, 6) and np.isfinite(logs[0].points(i)[:, 5]).all()
    _same_all(logs[0], logs[1], n)


# ---- 3. tolerance mode -----------------------------------------------------------------------------------------------------------
def test_tolerance_points_within_1e4_db_of_exact():
    """5120 instances (10240 channels): with the plane off the fused K-weighting + true-peak kernel would run in tolerance mode"""
    import meters_lv2_b200 as B
    n = 5120
    fma, exact, fused = (B.EBUr128(n, 48000.0, True) for _ in range(3))
    for bank, prec in ((fma, B.PREC_FMA), (exact, B.PREC_EXACT), (fused, B.PREC_FMA)):
        bank.set_precision(prec)
        bank.control(bank.START)
    fma.log_enable(128, dbtp=True); exact.log_enable(128, dbtp=True); fused.log_enable(128)
    base = torch.from_numpy(sig(2 * n, 0, 4096, seed=4)).cuda()
    for b in range(110):
        s = (b * 1024) % 3072
        x = base[:, s:s + 1024] * (0.25 + 0.75 * ((b // 7) % 4) / 3)
        if 30 <= b < 60:
            x = x.clone(); x[0::14] = 0.0; x[1::14] = 0.0  # instances 0, 7, 14 ... fall silent: their whole fragments read -inf
        d = []
        for bank in (fma, exact, fused):
            torch.cuda.synchronize()
            l0 = B.launch_count(); bank.run(x); d.append(B.launch_count() - l0)
        # K1 + the chunk-parallel true-peak kernel + the fold in place of the fused kernel
        assert d[0] == d[1] and d[0] - d[2] == 2, (b, d)
    logs = [_Acc(n), _Acc(n)]
    for acc, bank in zip(logs, (fma, exact)):
        acc.drain(bank)
    ninf = 0
    for i in range(n):
        a, e = logs[0].points(i)[:, 5], logs[1].points(i)[:, 5]
        assert np.array_equal(np.isneginf(a), np.isneginf(e)), i
        ninf += int(np.isneginf(e).sum())
        sel = e > -120.0
        assert np.all(np.abs(a[sel].astype(np.float64) - e[sel]) <= 1e-4), (i, np.max(np.abs(a[sel] - e[sel])))
        assert np.array_equal(u32(logs[0].points(i)[:, :5]), u32(logs[1].points(i)[:, :5])), i
    assert ninf > 0


# ---- 4. the hold invariant at scale ----------------------------------------------------------------------------------------------
def test_points_fold_to_the_hold_at_8192():
    import meters_lv2_b200 as B
    n, nf = 8192, 1024
    bank = B.EBUr128(n, 48000.0, True)
    bank.log_enable(64, dbtp=True)
    bank.control(bank.START)
    g = torch.Generator(device="cuda").manual_seed(1)
    base = torch.rand(2 * n, 4 * nf, device="cuda", generator=g) * 2 - 1
    lvl = torch.rand(n, 16, device="cuda", generator=g).repeat_interleave(2, 0) ** 3
    for b in range(75):                                    # 76800 frames: exactly 32 fragments
        s = (b % 4) * nf
        bank.run(base[:, s:s + nf] * lvl[:, (b // 9) % 16, None])
    pts, cnt, lost = bank.log_drain()
    _, tp = bank.results()
    assert (cnt == 32).all() and not lost.any()
    assert np.array_equal(u32(pts["dbtp"][:, :32].max(axis=1)), u32(tp))
    bank.run(base[:, :nf] * 3.0)                           # 1024 frames into a fragment: the louder frames are in no point yet
    _, cnt2, _ = bank.log_drain()
    _, tp2 = bank.results()
    assert (cnt2 == 0).all()
    assert np.all(pts["dbtp"][:, :32].max(axis=1) < tp2)


# ---- 5. restore: the open fragment restarts ---------------------------------------------------------------------------------------
def test_restore_drops_the_open_fragment():
    import meters_lv2_b200 as B
    n, nf = 12, 1000
    a = B.EBUr128(n, 48000.0, True)
    a.log_enable(256, dbtp=True); a.control(a.START)
    orc_a, orc_b = _TpOracle(n, 2), _TpOracle(n, 2)
    for blk in range(13):                                  # 13000 frames: 5 fragments and 1000 frames into the 6th
        x = sig(2 * n, blk * nf, nf, seed=6)
        a.run(torch.from_numpy(x).cuda())
        orc_a.process(x); orc_b.process(x)
    snap = a.snapshot()
    b = B.EBUr128(n, 48000.0, True)
    b.log_enable(256, dbtp=True)
    b.restore(snap)
    a.log_drain()                                          # the points before the snapshot
    for i in range(n):
        orc_b.cut(i)
    orc_a.pts = [[] for _ in range(n)]
    orc_b.pts = [[] for _ in range(n)]
    for blk in range(13, 40):
        x = sig(2 * n, blk * nf, nf, seed=6)
        for bank in (a, b):
            bank.run(torch.from_numpy(x).cuda())
        orc_a.process(x); orc_b.process(x)
    acc_a, acc_b = _Acc(n), _Acc(n)
    acc_a.drain(a); acc_b.drain(b)
    _same_tp(acc_a, orc_a, range(n), "kept")
    _same_tp(acc_b, orc_b, range(n), "restored")
    # the loudness fields, and every dBTP point after the first, are the same in both banks
    _same_all(acc_a, acc_b, n, 5)
    for i in range(n):
        assert np.array_equal(u32(acc_a.points(i)[1:, 5]), u32(acc_b.points(i)[1:, 5])), i


# ---- 6. programme_loudness(curves=True) -------------------------------------------------------------------------------------------
def test_programme_loudness_curve_tp():
    import meters_lv2_b200 as B
    fs, fragm, block = 48000.0, 2400, 1024
    lengths = np.array([0, 1000, 7 * fragm, 3 * 60 * 48000 + 777, 50 * fragm + 123, fragm, 95 * fragm], np.int64)
    n = lengths.size
    get = lambda off, m: sig(2 * n, off, m, seed=5)
    out = B.programme_loudness(get, lengths, fs, block=block, curves=True)
    ref = B.programme_loudness(get, lengths, fs, block=block)
    for k, v in ref.items():
        assert np.array_equal(np.asarray(out[k]).view(np.uint32), np.asarray(v).view(np.uint32)), k
    c = out["curve_TP"]
    assert c.dtype == np.float32 and c.shape == (n, int((lengths // fragm).max()))
    orc = _TpOracle(n, 2, fs)
    total = int(lengths.max())
    for off in range(0, total, block):
        m = min(block, total - off)
        orc.process(get(off, m), lens=np.clip(lengths - off, 0, m))
    for i in range(n):
        npt = int(lengths[i] // fragm)
        assert np.array_equal(u32(c[i, :npt]), u32(orc.points(i))), i
        assert np.isnan(c[i, npt:]).all(), i
    off = B.programme_loudness(lambda o, m: sig(6, o, m, seed=5), lengths[[1, 2, 5]], fs, block=block, dbtp=False, curves=True)
    assert np.isneginf(off["curve_TP"][[1, 2], :off["n_points"][[1, 2]].min()]).all()
    assert np.isneginf(off["curve_TP"][1, :7]).all() and np.isnan(off["curve_TP"][0]).all()


# ---- 7. error codes and the low-rate limit ----------------------------------------------------------------------------------------
def test_log_errors_are_codes():
    import meters_lv2_b200 as B
    L = B.lib()
    n = 256
    bank = B.EBUr128(n, 48000.0, True)
    pts = np.empty((n, 8), B.R128_POINT_DTYPE); cnt = np.empty(n, np.uint32); lost = np.empty(n, np.uint64)
    args = (B._np_ptr(pts), B._np_ptr(cnt), B._np_ptr(lost), None)
    assert L.b200m_r128_log_drain(bank.h, *args) == -1                # no log
    bank.log_enable(8)
    assert L.b200m_r128_log_drain(bank.h, *args) == -1                # a loudness-only log
    assert L.b200m_r128_log_enable(None, 8, None) == -1
    assert L.b200m_r128_log_drain(None, *args) == -1
    assert L.b200m_r128_log_enable(bank.h, 8, None) == 0
    assert L.b200m_r128_log_drain(bank.h, None, *args[1:]) == -1
    x = torch.from_numpy(sig(2 * n, 0, 4800)).cuda()
    bank.control(bank.START)
    bank.run(x)
    assert L.b200m_r128_log_drain(bank.h, *args) == 0 and (cnt == 2).all() and np.isfinite(pts["dbtp"][:, :2]).all()
    # b200m_ebu_log_enable on the member bank: a loudness-only log again
    assert L.b200m_ebu_log_enable(bank.ebu.h, 8, None) == 0
    assert L.b200m_r128_log_drain(bank.h, *args) == -1
    bank.run(x)
    p5, c5, _ = bank.ebu.log_drain()
    assert p5.dtype == B.EBU_POINT_DTYPE and (c5 == 2).all()
    # capacity 0 turns both off
    assert L.b200m_r128_log_enable(bank.h, 8, None) == 0
    assert L.b200m_r128_log_enable(bank.h, 0, None) == 0
    assert L.b200m_ebu_log_capacity(bank.ebu.h) == 0
    assert L.b200m_r128_log_drain(bank.h, *args) == -1
    with pytest.raises(B.B200MError, match="log is off"):
        bank.ebu.log_drain()
    # no device can hold it: B200M_E_NOMEM, both off, and the bank keeps working
    assert L.b200m_r128_log_enable(bank.h, C.c_uint32(0xFFFFFFFF), None) == -2
    assert L.b200m_r128_log_drain(bank.h, *args) == -1
    bank.run(x)
    assert np.isfinite(bank.results()[1]).all()
    # below 5120 Hz (fragments of < 256 frames) the plane is refused, the loudness log is not
    low = B.EBUr128(8, 4800.0, True)
    assert L.b200m_r128_log_enable(low.h, 16, None) == -4
    assert L.b200m_ebu_log_capacity(low.ebu.h) == 0
    low.log_enable(16)
    assert L.b200m_ebu_log_capacity(low.ebu.h) == 16


def test_lowest_rate_with_fragments_of_one_chunk():
    """5120 Hz: 256-frame fragments, one true-peak chunk each, up to 33 edges in an 8192-frame block"""
    import meters_lv2_b200 as B
    fs, n, nf = 5120.0, 8, 8192
    bank = B.EBUr128(n, fs, True)
    bank.set_precision(B.PREC_EXACT)
    bank.log_enable(200, dbtp=True)
    bank.control(bank.START)
    orc = _TpOracle(n, 2, fs)
    acc = _Acc(n)
    for b in range(8):
        if b == 3:
            bank.control(bank.NEW, 5); orc.new(5)
        m = nf if b % 2 == 0 else 8192 - 77
        x = sig(2 * n, b * nf, m, seed=12, fs=fs)
        bank.run(torch.from_numpy(x).cuda())
        orc.process(x)
        acc.drain(bank)
    _same_tp(acc, orc, range(n))
