"""GPU: the window log of the DR-14 bank (b200m_dr14_log_enable / b200m_dr14_log_drain) and programme_dr14(curves=True).

Every bank instance has a private reference dr14 plugin (_oracle.Dr14, the reference build when present) fed the same frames and
read after every block in which one of its 3 s windows closed: a point's m_rms, dr, dr_total and block_count must equal those
ports bit for bit.  A point's own window values (rms, peak), its second-highest window peak and its silent flag are restated here
with numpy: a float32 sequential sum per window, the reference's expression types, and coeff_to_db through the host libm's log10f.
"""
import ctypes as C
import ctypes.util

import numpy as np
import pytest
import torch

import _oracle as O

pytestmark = pytest.mark.gpu
F32 = np.float32
NAN = F32(np.nan)
_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.log10f.restype = C.c_float
_libm.log10f.argtypes = [C.c_float]
FILL = (np.nan, np.inf, -np.inf, 1e30)


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def db(c):
    """coeff_to_db (src/dr14.c:236-239) with the host libm"""
    c = F32(c)
    return F32(-80.0) if float(c) < .0001 else F32(F32(20.0) * F32(_libm.log10f(c)))


def _win(rate):
    return int(np.rint(F32(rate * 3.0))) + 1


class _Restate:
    """one instance's window sums, peaks and second-peak pair as dr14_run keeps them (:401-416, :285-352), in numpy"""

    def __init__(self, nch, rate):
        self.nch, self.nsc = nch, F32(np.rint(F32(rate * 3.0)))
        self.w = int(self.nsc) + 1
        self.reset()

    def reset(self):
        self.s = np.zeros(self.nch, F32); self.pc = np.zeros(self.nch, F32); self.h = np.zeros((self.nch, 2), F32)
        self.nf = 0; self.win = 0; self.cnt = 0
        self.peak2 = np.full(self.nch, -81.0, F32)

    def _acc(self, seg):
        if seg.shape[1] == 0:
            return
        sq = (seg * seg).astype(F32)
        self.s = np.add.accumulate(np.concatenate([self.s[:, None], sq], axis=1), axis=1)[:, -1].astype(F32)
        self.pc = np.maximum(self.pc, seg.max(axis=1)).astype(F32)

    def feed(self, xi):
        """xi [nch, L]: the point of the window that closes in it (a dict without the running fields), or None"""
        k = self.w - self.cnt
        if xi.shape[1] < k:
            self._acc(xi)
            self.cnt += xi.shape[1]
            return None
        self._acc(xi[:, :k])
        p = self._close()
        self._acc(xi[:, k:])
        self.cnt = xi.shape[1] - k
        return p

    def _close(self):
        self.win += 1
        silent = not any(float(v) > 1e-9 * float(self.nsc) for v in self.s)
        if silent:
            self.s[:] = 0
            return dict(window=self.win, silent=True, rms=[F32(-80.0)] * self.nch, peak=[NAN] * self.nch, peak2=self.peak2.copy())
        self.nf += 1
        rms = [db(F32(np.sqrt(np.float64(F32(F32(F32(2.0) * self.s[c]) / self.nsc))))) for c in range(self.nch)]
        peak = [db(self.pc[c]) for c in range(self.nch)]
        for c in range(self.nch):
            pc = self.pc[c]
            if pc >= self.h[c, 0]:
                self.h[c, 1] = self.h[c, 0]; self.h[c, 0] = pc
            elif pc > self.h[c, 1]:
                self.h[c, 1] = pc
        self.pc[:] = 0; self.s[:] = 0
        self.peak2 = np.array([db(self.h[c, 1]) if self.nf > 2 else -81.0 for c in range(self.nch)], F32)
        return dict(window=self.win, silent=False, rms=rms, peak=peak, peak2=self.peak2.copy())


def _point(p, ref_row, nch):
    """the expected b200m_dr14_point from a restated window and the reference's ports read after its block"""
    import meters_lv2_b200 as B
    e = np.zeros((), B.DR14_POINT_DTYPE)
    e["window"] = p["window"]; e["silent"] = 1.0 if p["silent"] else 0.0
    for f in ("rms", "peak", "m_rms", "peak2", "dr"):
        e[f] = NAN
    e["rms"][:nch] = p["rms"]; e["peak"][:nch] = p["peak"]; e["peak2"][:nch] = p["peak2"]
    e["m_rms"][:nch] = ref_row[6:6 + nch]; e["dr"][:nch] = ref_row[8:8 + nch]
    e["dr_total"] = ref_row[10] if nch == 2 else NAN
    e["block_count"] = ref_row[11]
    return e


class _Priv:
    """private instances: a reference plugin and a restatement per bank instance, and the points they expect"""

    def __init__(self, n, nch, rate):
        self.n, self.nch, self.rate = n, nch, rate
        self.ref = [O.Dr14(1, nch, rate, True) for _ in range(n)]
        self.rs = [_Restate(nch, rate) for _ in range(n)]
        self.want = [[] for _ in range(n)]

    def feed(self, x, lens=None):
        """one block: x [n * nch, nfram], instance i over its first lens[i] frames; the instances whose window closed"""
        closed = []
        for i in range(self.n):
            L = x.shape[1] if lens is None else int(lens[i])
            if L == 0:
                continue
            xi = np.ascontiguousarray(x[i * self.nch:(i + 1) * self.nch, :L])
            self.ref[i].process(xi)
            p = self.rs[i].feed(xi)
            if p is not None:
                self.want[i].append(_point(p, self.ref[i].read()[0], self.nch))
                closed.append(i)
        return closed

    def reset(self, i):
        self.ref[i].reset(); self.rs[i].reset()

    def clear(self, i):
        self.ref[i] = O.Dr14(1, self.nch, self.rate, True); self.rs[i].reset()


class _Acc:
    """the drained points of every instance, concatenated over drains"""

    def __init__(self, n):
        self.p = [[] for _ in range(n)]

    def drain(self, bank, stream=None):
        pts, cnt, lost = bank.log_drain(stream)
        assert not lost.any()
        assert np.isnan(pts["window"][np.arange(pts.shape[1])[None, :] >= cnt[:, None].astype(np.int64)]).all()
        for i in range(pts.shape[0]):
            self.p[i].extend(pts[i, :cnt[i]])
        return pts, cnt


def _check(acc, priv, tag=""):
    for i in range(priv.n):
        got, want = acc.p[i], priv.want[i]
        assert len(got) == len(want), (tag, i, len(got), len(want))
        for k, (g, w) in enumerate(zip(got, want)):
            assert g.tobytes() == w.tobytes(), (tag, i, k, g, w)


def _music(rows, n, seed):
    """noise under a slow loudness envelope, different per row"""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    ph = rng.uniform(0, 6.28, (rows, 1))
    per = rng.uniform(5000, 90000, (rows, 1))
    env = (0.05 + 0.95 * np.abs(np.sin(2 * np.pi * t / per + ph))).astype(np.float32)
    g = rng.uniform(0.05, 0.9, (rows, 1)).astype(np.float32)
    return (rng.uniform(-1, 1, (rows, n)).astype(np.float32) * env * g).astype(np.float32)


def _click(rate):
    """a click whose square is half the silence gate's threshold 1e-9 * n_sample_cnt (:290)"""
    return F32(np.sqrt(0.5e-9 * np.rint(F32(rate * 3.0))))


def _signal(n, nch, rate, nwin, seed):
    """music-like noise with stretches of digital silence: instance i's windows j and j + 1 (j = 2 + i % 3, counted from 0) are
    all zero but for a positive click in the second (still under the silence gate), and window j + 2 is quiet, so the carried
    click is its peak; nwin >= 7"""
    w = _win(rate)
    x = _music(n * nch, nwin * w + w // 2, seed)
    for i in range(n):
        r = slice(i * nch, (i + 1) * nch)
        a = (2 + i % 3) * w
        x[r, a:a + 2 * w] = 0.0
        x[r, a + w + 777] = _click(rate)
        x[r, a + 2 * w:a + 3 * w] *= F32(0.4) * _click(rate) / np.abs(x[r, a + 2 * w:a + 3 * w]).max()
    return x


@pytest.mark.parametrize("block", [1024, 8192, 1000])
@pytest.mark.parametrize("rate", [48000.0, 44100.0])
@pytest.mark.parametrize("nch", [2, 1])
def test_dr14_log_parity(nch, rate, block):
    """every point against the reference and the restatement; each scored window's bin is the one the histogram gained"""
    import meters_lv2_b200 as B
    n, nwin = 3, 9
    x = _signal(n, nch, rate, nwin, seed=int(rate) + nch + block)
    bank = B.DR14(n, nch, rate, True)
    bank.log_enable(32)
    priv = _Priv(n, nch, rate)
    acc = _Acc(n)
    before = [[bank.histogram(i, c) for c in range(nch)] for i in range(n)]
    for off in range(0, x.shape[1], block):
        xb = np.ascontiguousarray(x[:, off:off + block])
        bank.run(torch.from_numpy(xb).cuda())
        for i in priv.feed(xb):
            p = priv.want[i][-1]
            for c in range(nch):
                h = bank.histogram(i, c)
                gained = np.nonzero(h != before[i][c])[0]
                if p["silent"] == 0:
                    b = int(np.rint(F32(F32(100.0) * F32(F32(80.0) + p["rms"][c])))) - 1
                    b = min(b, 7999)
                    want = [b] if b > 0 else []
                    assert gained.tolist() == want and all(h[gained] == before[i][c][gained] + 1), (off, i, c, gained, b)
                else:
                    assert gained.size == 0
                before[i][c] = h
    acc.drain(bank)
    _check(acc, priv)
    for i in range(n):
        pts = acc.p[i]
        assert [int(p["window"]) for p in pts] == list(range(1, nwin + 1))
        j = 2 + i % 3
        assert [int(p["silent"]) for p in pts] == [int(k in (j, j + 1)) for k in range(nwin)]
        # the click of the silent window is the next scored window's peak
        assert pts[j + 2]["peak"][0] == db(_click(rate))


def _ragged_lengths(rng, n, nfram, priv):
    pool = np.array([0, 1, 2, 47, nfram, nfram, nfram])
    lens = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, nfram + 1, n))
    for i in range(n):
        left = priv.rs[i].w - priv.rs[i].cnt
        if left <= nfram:
            u = rng.random()
            lens[i] = left if u < 0.3 else left - 1 if u < 0.5 else 0 if u < 0.6 else lens[i]
    return np.minimum(lens, nfram).astype(np.uint32)


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_dr14_log_ragged(host):
    """ragged blocks: a window is logged only if it closes within the instance's own frames; NaN / Inf after them"""
    import meters_lv2_b200 as B
    n, nch, rate = 6, 2, 8000.0
    rng = np.random.default_rng(3)
    sizes = rng.integers(1, 8193, 260)
    x_all = _music(n * nch, int(sizes.sum()), 21)
    x_all[2 * nch:3 * nch, 50000:200000] = 0.0                    # silent windows on instance 2
    bank = B.DR14(n, nch, rate, True)
    bank.log_enable(64)
    priv = _Priv(n, nch, rate)
    acc = _Acc(n)
    t = 0
    for b, nf in enumerate(sizes):
        nf = int(nf)
        lens = _ragged_lengths(rng, n, nf, priv)
        x = x_all[:, t:t + nf].copy()
        for i in range(n):
            x[i * nch:(i + 1) * nch, lens[i]:] = FILL[(b + i) % len(FILL)]
        bank.run(x if host else torch.from_numpy(x).cuda(), lengths=lens)
        priv.feed(x, lens)
        t += nf
    acc.drain(bank)
    _check(acc, priv)
    assert min(len(p) for p in priv.want) >= 5 and any(int(p["silent"]) for p in priv.want[2])


def _curves_want(x, lens, nch, rate, block):
    """per track the points a private reference instance and restatement give, fed in blocks of `block` frames"""
    out = []
    for i, L in enumerate(lens):
        pr = _Priv(1, nch, rate)
        for off in range(0, int(L), block):
            pr.feed(np.ascontiguousarray(x[i * nch:(i + 1) * nch, off:min(int(L), off + block)]))
        out.append(pr.want[0])
    return out


def _check_curves(res, cv, want, lens, nch, rate):
    w = _win(rate)
    assert np.array_equal(cv["n_windows"], np.asarray(lens) // w)
    W = int(cv["n_windows"].max())
    for k in ("window_rms", "window_peak", "m_rms", "peak2", "dr"):
        assert cv[k].shape == (len(lens), W, nch) and cv[k].dtype == np.float32
    assert cv["dr_total"].shape == cv["block_count"].shape == cv["silent"].shape == (len(lens), W)
    for i, pts in enumerate(want):
        m = len(pts)
        assert m == cv["n_windows"][i]
        for j, p in enumerate(pts):
            for k, f in (("window_rms", "rms"), ("window_peak", "peak"), ("m_rms", "m_rms"), ("peak2", "peak2"), ("dr", "dr")):
                assert u32(cv[k][i, j]).tolist() == u32(p[f][:nch]).tolist(), (i, j, k)
            for k in ("dr_total", "block_count"):
                assert u32(cv[k][i, j]) == u32(p[k]), (i, j, k)
            assert cv["silent"][i, j] == bool(p["silent"])
        for k in ("window_rms", "window_peak", "m_rms", "peak2", "dr", "dr_total", "block_count"):
            assert np.isnan(cv[k][i, m:]).all()
        assert not cv["silent"][i, m:].any()


@pytest.mark.parametrize("form", ["host", "device", "callable"])
def test_programme_dr14_curves(form):
    import meters_lv2_b200 as B
    rate, nch, n, block = 8000.0, 2, 12, 1024
    w = _win(rate)
    rng = np.random.default_rng(31)
    lens = rng.integers(0, 40 * w, n)
    lens[:5] = [0, w - 1, w, 3 * w + 5, 41 * w]                    # empty, shorter than a window, exactly one, and 41 windows
    x = _music(n * nch, int(lens.max()), 32)
    x[3 * nch:4 * nch, w:3 * w] = 0.0
    for i in range(n):                                             # frames past a track's end are never read
        x[i * nch:(i + 1) * nch, lens[i]:] = FILL[i % len(FILL)]
    if form == "host":
        arg = x
    elif form == "device":
        arg = torch.from_numpy(x).cuda()
    else:
        def arg(off, nfram):
            return torch.from_numpy(np.ascontiguousarray(x[:, off:off + nfram])).cuda()
    res, cv = B.programme_dr14(arg, lens, rate, nch, True, block=block, curves=True)
    plain = B.programme_dr14(x, lens, rate, nch, True, block=block)
    assert res.tobytes() == plain.tobytes()
    _check_curves(res, cv, _curves_want(x, lens, nch, rate, block), lens, nch, rate)


def test_programme_dr14_curves_mono_and_errors():
    import meters_lv2_b200 as B
    rate, nch = 48000.0, 1
    w = _win(rate)
    lens = np.array([7 * w + 3, 2 * w, 0])
    x = _music(3, int(lens.max()), 33)
    res, cv = B.programme_dr14(x, lens, rate, nch, True, block=8192, curves=True)
    _check_curves(res, cv, _curves_want(x, lens, nch, rate, 8192), lens, nch, rate)
    assert res.tobytes() == B.programme_dr14(x, lens, rate, nch, True, block=8192).tobytes()
    with pytest.raises(B.B200MError):
        B.programme_dr14(x, lens, rate, nch, False, curves=True)


FORMS = {"fused": {}, "wide": {"B200M_TPK_WIDE": "2", "B200M_TPK_SPLIT": "0"},
         "slabs": {"B200M_TPK_SPLIT": "2", "B200M_TPK_SLAB": "192"}}


def test_dr14_log_forms_and_paths(monkeypatch):
    """the fused, wide and slab process() forms, on the host and the device path, log the same bits"""
    import meters_lv2_b200 as B
    n, nch, rate, nwin = 24, 2, 8000.0, 8
    w = _win(rate)
    x = _signal(n, nch, rate, nwin, seed=5)
    x[:, 6 * w + 100] = np.nan                                     # a NaN sum is gated as silent too
    logs = {}
    for form, env in FORMS.items():
        for host in (False, True):
            with monkeypatch.context() as mp:
                for k, v in env.items():
                    mp.setenv(k, v)
                bank = B.DR14(n, nch, rate, True)
            bank.log_enable(16)
            for off in range(0, x.shape[1], 1024):
                xb = np.ascontiguousarray(x[:, off:off + 1024])
                bank.run(xb if host else torch.from_numpy(xb).cuda())
            pts, cnt, lost = bank.log_drain()
            assert (cnt == nwin).all() and not lost.any()
            logs[form, host] = pts.tobytes()
            bank.close()
    assert len(set(logs.values())) == 1
    pts = np.frombuffer(logs["fused", False], B.DR14_POINT_DTYPE).reshape(n, 16)
    assert (pts["silent"][:, 6] == 1).all() and (pts["rms"][:, 6] == -80).all() and np.isnan(pts["peak"][:, 6]).all()
    assert (pts["silent"][:, :nwin].sum(axis=1) == 3).all()


def test_dr14_log_controls():
    """RESET / CLEAR mid-window and before the block in which the window would close: no point for the dropped window, the
    count restarts at 1, the other instances and the points already logged are untouched"""
    import meters_lv2_b200 as B
    n, nch, rate, block = 6, 2, 8000.0, 1000
    w = _win(rate)
    x = _music(n * nch, 12 * w - 10, 41)
    bank = B.DR14(n, nch, rate, True)
    bank.log_enable(32)
    priv = _Priv(n, nch, rate)
    acc = _Acc(n)
    # instance 1 mid-window, instance 2 in the block in which its 3rd window would close, instance 3 cleared there
    ctl = {30: [(B.DR14_RESET, [1])], (3 * w) // block: [(B.DR14_RESET, [2]), (B.DR14_CLEAR, [3])], 150: [(B.DR14_RESET, [1, 4])]}
    for b, off in enumerate(range(0, x.shape[1], block)):
        for cmd, inst in ctl.get(b, []):
            bank.control(cmd, inst)
            for i in inst:
                priv.reset(i) if cmd == B.DR14_RESET else priv.clear(i)
        xb = np.ascontiguousarray(x[:, off:off + block])
        bank.run(torch.from_numpy(xb).cuda())
        priv.feed(xb)
        if b == 60:
            acc.drain(bank)
    acc.drain(bank)
    _check(acc, priv)
    win = [[int(p["window"]) for p in acc.p[i]] for i in range(n)]
    assert win[0] == list(range(1, 12)) and win[5] == win[0]
    assert win[2][:2] == [1, 2] and win[2][2] == 1 and win[3][2] == 1
    assert 1 in win[1][1:] and win[4].count(1) == 2
    # enabling again empties the log; capacity 0 turns it off
    bank.log_enable(8)
    pts, cnt, lost = bank.log_drain()
    assert not cnt.any() and not lost.any() and pts.shape == (n, 8)
    bank.log_enable(0)
    assert B.lib().b200m_dr14_log_capacity(bank.h) == 0
    with pytest.raises(B.B200MError):
        bank.log_drain()


def test_dr14_log_changes_nothing_else():
    import meters_lv2_b200 as B
    n, nch, rate = 16, 2, 8000.0
    x = torch.from_numpy(_signal(n, nch, rate, 7, seed=9)).cuda()
    banks = [B.DR14(n, nch, rate, True) for _ in range(2)]
    banks[1].log_enable(8)
    for off in range(0, x.shape[1], 1024):
        d = []
        for bk in banks:
            c0 = B.launch_count()
            bk.run(x[:, off:off + 1024])
            d.append(B.launch_count() - c0)
        assert d[0] == d[1]
        assert banks[0].results().tobytes() == banks[1].results().tobytes()
    for i in range(n):
        for c in range(nch):
            assert np.array_equal(banks[0].histogram(i, c), banks[1].histogram(i, c))
    assert (banks[1].log_drain()[1] == 7).all()


def test_dr14_log_overflow():
    import meters_lv2_b200 as B
    n, nch, rate = 4, 2, 8000.0
    w = _win(rate)
    x = torch.from_numpy(_music(n * nch, 7 * w + 10, 51)).cuda()
    bank = B.DR14(n, nch, rate, True)
    bank.log_enable(3)
    for off in range(0, x.shape[1], 4096):
        bank.run(x[:, off:off + 4096])
    pts, cnt, lost = bank.log_drain()
    assert (cnt == 3).all() and (lost == 4).all()
    assert (pts["window"] == np.array([5, 6, 7], np.float32)).all()
    assert (pts["block_count"][:, -1] == bank.results()["block_count"]).all()


def test_dr14_log_scale():
    """8192 stereo instances over 45 s, windows staggered by resets: at each drain the newest point is results()"""
    import meters_lv2_b200 as B
    n, nch, rate, block = 8192, 2, 48000.0, 1024
    w = _win(rate)
    bank = B.DR14(n, nch, rate, True)
    bank.log_enable(4)
    gen = torch.Generator(device="cuda")
    nblk = 45 * 48000 // block
    seen = np.zeros(n, np.int64)
    for b in range(nblk):
        if b == 40:
            bank.control(B.DR14_RESET, np.arange(0, n, 3))
        gen.manual_seed(b)
        env = 0.05 + torch.rand((n * nch, 1), device="cuda", generator=gen)
        bank.run(((torch.rand((n * nch, block), device="cuda", generator=gen) * 2 - 1) * env).contiguous())
        if (b * block) % w > ((b + 1) * block) % w or (b >= 40 and ((b - 40) * block) % w > ((b - 39) * block) % w):
            res = bank.results()
            pts, cnt, lost = bank.log_drain()
            assert not lost.any()
            i = np.nonzero(cnt)[0]
            assert i.size
            last = pts[i, cnt[i].astype(np.int64) - 1]
            for f in ("m_rms", "dr", "dr_total", "block_count"):
                assert u32(last[f]).tobytes() == u32(res[f][i]).tobytes(), (b, f)
            seen[i] += cnt[i]
    assert seen.min() >= 13


def test_dr14_log_ordering():
    """a drain right behind run_host sees that block's window; so does one on the caller's stream after a device-path run"""
    import meters_lv2_b200 as B
    n, nch, rate = 64, 2, 8000.0
    w = _win(rate)
    x = _music(n * nch, w + 8, 61)
    cuts = [0, 8000, 16000, w - 1, w + 8]                          # the window closes on the last block's first frame
    bank = B.DR14(n, nch, rate, True)
    bank.log_enable(4)
    for a, b in zip(cuts[:-1], cuts[1:]):
        bank.run(np.ascontiguousarray(x[:, a:b]))
    pts, cnt, _ = bank.log_drain()
    assert (cnt == 1).all() and (pts["window"][:, 0] == 1).all()
    s = torch.cuda.Stream()
    xd = torch.from_numpy(x).cuda()
    bank2 = B.DR14(n, nch, rate, True)
    bank2.log_enable(4)
    with torch.cuda.stream(s):
        for a, b in zip(cuts[:-2], cuts[1:-1]):
            bank2.run(xd[:, a:b], stream=s)
        torch.cuda._sleep(5_000_000)                              # the last block is still queued when the drain is called
        bank2.run(xd[:, w - 1:], stream=s)
        pts2, cnt2, _ = bank2.log_drain(stream=s)
    assert (cnt2 == 1).all()
    assert pts2[:, :1].tobytes() == pts[:, :1].tobytes()


def test_dr14_log_errors():
    import meters_lv2_b200 as B
    L = B.lib()
    INVAL, NOMEM, UNSUPPORTED = -1, -2, -4
    tp = B.DR14(4, 2, 48000.0, False)
    assert L.b200m_dr14_log_enable(tp.h, 8, None) == UNSUPPORTED
    with pytest.raises(B.B200MError):
        tp.log_enable(8)
    bank = B.DR14(4, 2, 48000.0, True)
    cnt = np.empty(4, np.uint32); lost = np.empty(4, np.uint64); pts = np.empty((4, 1), B.DR14_POINT_DTYPE)
    assert L.b200m_dr14_log_drain(bank.h, B._np_ptr(pts), B._np_ptr(cnt), B._np_ptr(lost), None) == INVAL    # the log is off
    assert L.b200m_dr14_log_enable(None, 8, None) == INVAL
    assert L.b200m_dr14_log_capacity(None) == 0
    bank.log_enable(2)
    for args in ((None, B._np_ptr(cnt), B._np_ptr(lost)), (B._np_ptr(pts), None, B._np_ptr(lost)), (B._np_ptr(pts), B._np_ptr(cnt), None)):
        assert L.b200m_dr14_log_drain(bank.h, *args, None) == INVAL
    assert L.b200m_dr14_log_drain(None, B._np_ptr(pts), B._np_ptr(cnt), B._np_ptr(lost), None) == INVAL
    assert L.b200m_dr14_log_enable(bank.h, 0xFFFFFFFF, None) == NOMEM
    assert L.b200m_dr14_log_capacity(bank.h) == 0
    bank.run(torch.zeros(8, 64, device="cuda"))                  # the bank still runs, the failed allocation did not stick
    bank.log_enable(2)
    assert L.b200m_dr14_log_capacity(bank.h) == 2
