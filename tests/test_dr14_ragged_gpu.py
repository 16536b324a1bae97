"""GPU: ragged blocks of the DR-14 / TPnRMS bank (b200m_dr14_run_ragged_*) and programme_dr14.

Every bank instance i is compared with a private instance that sees only its own frames: one _oracle.Dr14 of one instance (the
reference dr14 plugin where oracle/_ref is built), fed the first len[i] frames of each block with len[i] > 0, and for the 8000-bin
histograms one plain DR14 bank of one instance fed the same frames.  Frames at or after len[i] hold NaN, +-Inf or 1e30.
"""
import ctypes as C

import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
# _oracle.Dr14.read() columns -> (result field, channel)
COLS = [("v_rms", 0), ("v_rms", 1), ("v_peak", 0), ("v_peak", 1), ("m_peak", 0), ("m_peak", 1), ("m_rms", 0), ("m_rms", 1),
        ("dr", 0), ("dr", 1), ("dr_total", None), ("block_count", None)]
FILL = (np.nan, np.inf, -np.inf, 1e30)


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _win(rate):
    return int(np.rint(np.float32(rate * 3.0))) + 1


def _music(rows, n, seed):
    """noise under a slow loudness envelope, different per row, so that the 3 s windows and the channels differ"""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    ph = rng.uniform(0, 6.28, (rows, 1))
    per = rng.uniform(5000, 90000, (rows, 1))
    env = (0.05 + 0.95 * np.abs(np.sin(2 * np.pi * t / per + ph))).astype(np.float32)
    g = rng.uniform(0.05, 0.9, (rows, 1)).astype(np.float32)
    return (rng.uniform(-1, 1, (rows, n)).astype(np.float32) * env * g).astype(np.float32)


class _Priv:
    """private instances: the reference plugin (results) and a plain bank of one (histograms, DR mode)"""

    def __init__(self, n, nch, rate, dr_mode, hist):
        import meters_lv2_b200 as B
        self.n, self.nch, self.rate, self.dr_mode, self.hist = n, nch, rate, dr_mode, hist
        self.ref = [O.Dr14(1, nch, rate, dr_mode) for _ in range(n)]
        self.one = [B.DR14(1, nch, rate, dr_mode) for _ in range(n)] if hist else None
        self.ran = np.zeros(n, bool)                  # ran since the last clear (a cleared, never-run plugin has no port values)
        self.cnt = np.zeros(n, np.int64)              # samples of the instance's current 3 s window

    def feed(self, x, lens):
        import torch
        for i in range(self.n):
            L = int(lens[i])
            if L == 0:
                continue
            xi = np.ascontiguousarray(x[i * self.nch:(i + 1) * self.nch, :L])
            self.ref[i].process(xi)
            if self.hist:
                self.one[i].run(torch.from_numpy(xi).cuda())
            self.ran[i] = True
            self.cnt[i] = (self.cnt[i] + L) % _win(self.rate)

    def reset(self, i):
        self.ref[i].reset()
        if self.hist:
            self.one[i].reset()
        self.cnt[i] = 0

    def clear(self, i):
        import meters_lv2_b200 as B
        self.ref[i] = O.Dr14(1, self.nch, self.rate, self.dr_mode)
        if self.hist:
            self.one[i] = B.DR14(1, self.nch, self.rate, self.dr_mode)
        self.ran[i] = False
        self.cnt[i] = 0

    def check(self, tag, got, bank=None):
        for i in range(self.n):
            if not self.ran[i]:
                continue
            want = self.ref[i].read()[0]
            for k, (f, c) in enumerate(COLS):
                if c is not None and c >= self.nch:
                    continue
                if f == "dr_total" and (self.nch == 1 or not self.dr_mode):
                    continue
                if f == "dr" and not self.dr_mode:
                    continue
                g = got[f][i] if c is None else got[f][i][c]
                assert u32(g) == u32(want[k]), (tag, i, f, c, g, want[k])
        if bank is not None and self.hist and self.dr_mode:
            for i in range(self.n):
                for c in range(self.nch):
                    assert np.array_equal(bank.histogram(i, c), self.one[i].histogram(0, c)), (tag, i, c)


def _sizes(nblk, seed):
    rng = np.random.default_rng(seed)
    s = rng.integers(1, 4097, nblk)
    s[[2, 17, 18, 101]] = 1
    s[[5, 6, 60, 150]] = 8192
    s[[30, 31, 80]] = 49
    return s


def _lengths(rng, n, nfram, priv):
    """random lengths with 0, 1..5, 47, 48, 49 and nfram; a few instances end on their window's last frame, one frame before it,
    or get 0 in the block where their window would close"""
    pool = np.array([0, 1, 2, 3, 4, 5, 47, 48, 49, nfram, nfram, nfram])
    lens = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, nfram + 1, n))
    w = _win(priv.rate)
    for i in range(n):
        left = w - int(priv.cnt[i])                   # the window closes on the instance's left-th next frame
        if left <= nfram:
            u = rng.random()
            if u < 0.25:
                lens[i] = left
            elif u < 0.45:
                lens[i] = left - 1
            elif u < 0.6:
                lens[i] = 0
    return np.minimum(lens, nfram).astype(np.uint32)


def _drive(bank, priv, x_all, sizes, seed, host, controls=None, zero_after=0):
    """feeds the bank and the private instances; controls {block: [(cmd, [inst, ...]), ...]} run before that block, and the first
    zero_after instances each control names get length 0 in that block"""
    import torch
    rng = np.random.default_rng(seed)
    n, nch = priv.n, priv.nch
    t = 0
    for b, nf in enumerate(sizes):
        nf = int(nf)
        if controls and b in controls:
            for cmd, inst in controls[b]:
                bank.control(cmd, inst)
                for i in inst:
                    priv.reset(i) if cmd == 1 else priv.clear(i)
        lens = _lengths(rng, n, nf, priv)
        if controls and b in controls:
            for _, inst in controls[b]:
                lens[inst[:zero_after]] = 0
        x = x_all[:, t:t + nf].copy()
        for i in range(n):                           # unread frames: NaN, +-Inf or 1e30
            x[i * nch:(i + 1) * nch, lens[i]:] = FILL[(b + i) % len(FILL)]
        bank.run(x if host else torch.from_numpy(x).cuda(), lengths=lens)
        priv.feed(x, lens)
        priv.check((b, nf), bank.results(), bank if b in (len(sizes) // 2, len(sizes) - 1) else None)
        t += nf
    return t


KINDS = {"dr14stereo": (True, 2), "dr14mono": (True, 1), "TPnRMSstereo": (False, 2), "TPnRMSmono": (False, 1)}


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("rate", [8000.0, 44100.0, 48000.0])
@pytest.mark.parametrize("kind", list(KINDS))
def test_dr14_ragged_parity(kind, rate, host):
    import meters_lv2_b200 as B
    dr_mode, nch = KINDS[kind]
    n = 6
    sizes = _sizes(300 if rate == 8000.0 else 200, 7)
    seed = int(rate) + nch + 10 * dr_mode + host
    x_all = _music(n * nch, int(sizes.sum()), seed)
    bank = B.DR14(n, nch, rate, dr_mode)
    priv = _Priv(n, nch, rate, dr_mode, hist=dr_mode)
    _drive(bank, priv, x_all, sizes, seed, host)
    if dr_mode and rate == 8000.0:
        assert min(r.read()[0][11] for r in priv.ref) > 0            # every instance scored windows


def test_dr14_ragged_controls():
    """per-instance RESET and CLEAR between ragged blocks, also on instances that get length 0 next"""
    import meters_lv2_b200 as B
    n, nch, rate = 8, 2, 8000.0
    sizes = _sizes(260, 3)
    x_all = _music(n * nch, int(sizes.sum()), 3)
    rng = np.random.default_rng(5)
    ctl = {}
    for b in range(10, 250, 9):
        ctl[b] = [(B.DR14_RESET if rng.random() < 0.6 else B.DR14_CLEAR, sorted(set(rng.integers(0, n, 3).tolist())))]
    bank = B.DR14(n, nch, rate, True)
    priv = _Priv(n, nch, rate, True, hist=True)
    _drive(bank, priv, x_all, sizes, 9, False, controls=ctl, zero_after=2)


@pytest.mark.parametrize("env", [{"B200M_TPK_SPLIT": "2"}, {"B200M_TPK_WIDE": "1"}], ids=["split", "wide"])
def test_dr14_ragged_opt_in_forms(env, monkeypatch):
    import meters_lv2_b200 as B
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n, nch, rate = 6, 2, 8000.0
    sizes = _sizes(160, 4)
    x_all = _music(n * nch, int(sizes.sum()), 4)
    bank = B.DR14(n, nch, rate, True)
    priv = _Priv(n, nch, rate, True, hist=True)
    _drive(bank, priv, x_all, sizes, 4, False)


@pytest.mark.parametrize("dr_mode", [True, False])
def test_dr14_ragged_uniform_is_plain(dr_mode):
    """all-nfram lengths and lengths=None are the plain call: same results, histograms and launches"""
    import torch
    import meters_lv2_b200 as B
    n, nch, rate = 64, 2, 8000.0
    sizes = _sizes(160, 6)
    x_all = torch.from_numpy(_music(n * nch, int(sizes.sum()), 6)).cuda()
    banks = [B.DR14(n, nch, rate, dr_mode) for _ in range(3)]
    t = 0
    for nf in sizes:
        nf = int(nf)
        xb = x_all[:, t:t + nf]
        d = []
        for k, bk in enumerate(banks):
            c0 = B.launch_count()
            if k == 0:
                bk.run(xb)
            elif k == 1:
                bk.run(xb, lengths=np.full(n, nf, np.uint32))
            else:
                p, s, rows, m = B._dev_ptr(xb)
                B._ck(B.lib().b200m_dr14_run_ragged_device(bk.h, p, s, m, None, B._stream_ptr(None)))
            d.append(B.launch_count() - c0)
        assert d[0] == d[1] == d[2], d
        r = [bk.results() for bk in banks]
        assert r[0].tobytes() == r[1].tobytes() == r[2].tobytes()
        t += nf
    if dr_mode:
        for i in (0, 17, 63):
            for c in range(nch):
                h = [bk.histogram(i, c) for bk in banks]
                assert np.array_equal(h[0], h[1]) and np.array_equal(h[0], h[2])


def test_dr14_ragged_invalid_lengths():
    import torch
    import meters_lv2_b200 as B
    n, nch = 4, 2
    bank = B.DR14(n, nch, 8000.0, True)
    x = torch.from_numpy(_music(n * nch, 30000, 8)).cuda()
    for off in range(0, 30000, 3000):
        bank.run(x[:, off:off + 3000], lengths=np.array([3000, 1000, 0, 2999], np.uint32))
    before = bank.results().tobytes(), [bank.histogram(i, c).copy() for i in range(n) for c in range(nch)]
    c0 = B.launch_count()
    bad = np.array([10, 11, 5, 3], np.uint32)
    p, s, rows, m = B._dev_ptr(x[:, :10])
    assert B.lib().b200m_dr14_run_ragged_device(bank.h, p, s, m, B._np_ptr(bad), B._stream_ptr(None)) == -1
    xh = np.ascontiguousarray(x[:, :10].cpu().numpy())
    ph, sh, _, mh = B._host_planar(xh)
    assert B.lib().b200m_dr14_run_ragged_host(bank.h, ph, sh, mh, B._np_ptr(bad)) == -1
    assert B.launch_count() == c0
    with pytest.raises(B.B200MError):
        bank.run(x[:, :10], lengths=[1, 2, 3])                     # wrong count
    assert bank.results().tobytes() == before[0]
    assert all(np.array_equal(a, b) for a, b in zip(before[1], [bank.histogram(i, c) for i in range(n) for c in range(nch)]))


def _private_track(x, L, nch, rate, dr_mode, block):
    """a private reference plugin fed one track in blocks of `block` frames with a short last block"""
    o = O.Dr14(1, nch, rate, dr_mode)
    for off in range(0, L, block):
        o.process(np.ascontiguousarray(x[:, off:min(L, off + block)]))
    return o.read()[0]


def _check_tracks(got, want, lens, nch, dr_mode):
    for i, w in enumerate(want):
        if lens[i] == 0:
            assert got[i].tobytes() == bytes(got.dtype.itemsize)
            continue
        for k, (f, c) in enumerate(COLS):
            if (c is not None and c >= nch) or (f == "dr_total" and (nch == 1 or not dr_mode)) or (f == "dr" and not dr_mode):
                continue
            g = got[f][i] if c is None else got[f][i][c]
            assert u32(g) == u32(w[k]), (i, lens[i], f, c, g, w[k])


def test_programme_dr14_stereo_tracks():
    import meters_lv2_b200 as B
    rate, nch, n = 44100.0, 2, 64
    w = _win(rate)
    rng = np.random.default_rng(12)
    lens = rng.integers(0, int(40 * rate) + 1, n)
    lens[:6] = [0, 3 * w, 5 * w, 7 * w, 1, w - 1]
    lens[6] = 9 * w + 100                                           # the silent track
    x = np.empty((n * nch, int(lens.max())), np.float32)
    for i in range(n):
        x[i * nch:(i + 1) * nch] = _music(nch, x.shape[1], 100 + i)[:, :]
    x[6 * nch:7 * nch] = 0.0
    got = B.programme_dr14(x, lens, rate, nch, True)
    want = [_private_track(x[i * nch:(i + 1) * nch], int(lens[i]), nch, rate, True, 1024) for i in range(n)]
    _check_tracks(got, want, lens, nch, True)
    assert got["block_count"][6] == 0.0 and got["dr_total"][6] == 21.0
    assert got["block_count"][1] == 9.0 and got["block_count"][2] == 15.0     # whole windows only


def test_programme_dr14_mono_tpnrms():
    import torch
    import meters_lv2_b200 as B
    rate, nch, n = 48000.0, 1, 16
    rng = np.random.default_rng(13)
    lens = rng.integers(0, int(20 * rate), n)
    lens[0] = 3
    x = _music(n, int(lens.max()), 13)
    got = B.programme_dr14(torch.from_numpy(x), lens, rate, nch, False, block=777)
    want = [_private_track(x[i:i + 1], int(lens[i]), nch, rate, False, 777) for i in range(n)]
    _check_tracks(got, want, lens, nch, False)


def test_programme_dr14_device_callable():
    import torch
    import meters_lv2_b200 as B
    rate, nch, n, block = 8000.0, 2, 512, 2048
    rng = np.random.default_rng(14)
    lens = rng.integers(0, int(15 * rate), n)
    lens[:3] = [0, _win(rate) * 3, 1]
    refs = [O.Dr14(1, nch, rate, True) for _ in range(n)]
    gen = torch.Generator(device="cuda")

    def f(off, nfram):
        gen.manual_seed(off)
        env = 0.1 + 0.9 * torch.sin(torch.arange(off, off + nfram, device="cuda", dtype=torch.float32) / 3000.0).abs()
        xb = ((torch.rand((n * nch, nfram), device="cuda", generator=gen) * 2 - 1) * env).contiguous()
        xh = xb.cpu().numpy()
        for i in range(n):                          # the private instances see each track's own frames only
            L = min(nfram, max(0, int(lens[i]) - off))
            if L:
                refs[i].process(np.ascontiguousarray(xh[i * nch:(i + 1) * nch, :L]))
        return xb

    got = B.programme_dr14(f, lens, rate, nch, True, block=block)
    _check_tracks(got, [r.read()[0] for r in refs], lens, nch, True)


def test_padding_changes_dr_ragged_does_not():
    """zero-padding a short track completes its partial last window, which is then scored; the ragged call never scores it"""
    import meters_lv2_b200 as B
    rate, nch = 8000.0, 2
    w = _win(rate)
    lens = np.array([3 * w + 2000, 6 * w + 17])
    x = _music(2 * nch, int(lens.max()), 15) * np.float32(4.0)
    got = B.programme_dr14(x, lens, rate, nch, True)
    want = [_private_track(x[i * nch:(i + 1) * nch], int(lens[i]), nch, rate, True, 1024) for i in range(2)]
    _check_tracks(got, want, lens, nch, True)
    xp = x.copy()
    xp[:nch, lens[0]:] = 0.0
    pad = B.programme_dr14(xp, np.full(2, lens.max()), rate, nch, True)
    assert pad[1].tobytes() == got[1].tobytes()
    assert pad["block_count"][0] != got["block_count"][0] or pad["dr_total"][0] != got["dr_total"][0] \
        or not np.array_equal(pad["m_peak"][0], got["m_peak"][0])
