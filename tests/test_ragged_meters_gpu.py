"""GPU: ragged blocks of the true-peak / K-meter, needle-meter, correlation and spectrum banks (b200m_*_process_ragged_*).

Every bank row group (a tpk channel, a needle unit, a correlation pair, a spectrum instance) is compared after every block with a
private _oracle instance of one meter fed only its own frames: the first len[i] frames of each block with len[i] > 0.  Frames at
or after len[i] hold NaN, +-Inf or 1e30.  Exact mode must match bit for bit, state and readings; tolerance mode stays within the
existing contracts (correlation 1e-5, spectrum and true-peak readings +-1e-4 dB).
"""
import ctypes as C

import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
FILL = (np.nan, np.inf, -np.inf, 1e30)
POOL = (0, 1, 3, 4, 5, 47, 48, 49, 63, 64, 65)
SIZES = (1024, 4097, 8192, 1024, 333, 4097, 64, 8192, 1000, 1024, 49, 4097)


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _db(v):
    return 20.0 * np.log10(np.maximum(np.abs(np.asarray(v, np.float64)), 1e-30))


def _signal(rows, n, seed):
    """noise under a per-row level and a slow envelope, so that the ballistics rise and fall within and across blocks"""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    env = np.abs(np.sin(2 * np.pi * t / rng.uniform(3000, 40000, (rows, 1)) + rng.uniform(0, 6.28, (rows, 1))))
    g = rng.uniform(0.02, 0.9, (rows, 1))
    return (rng.uniform(-1, 1, (rows, n)) * env * g).astype(np.float32)


def _lengths(rng, n, nfram, b, sit_out):
    """lengths 0, 1, 3, 4, 5, 47..49, 63..65, nfram - 1, nfram and random ones, new every block; the units in sit_out get 0 for
    blocks 3..6 (runs of skipped blocks)"""
    pool = np.array([p for p in POOL if p <= nfram] + [nfram - 1, nfram, nfram])
    ln = np.where(rng.random(n) < 0.6, rng.choice(pool, n), rng.integers(0, nfram + 1, n))
    if 3 <= b <= 6:
        ln[sit_out] = 0
    if (ln == nfram).all():
        ln[0] = nfram - 1
    return ln.astype(np.int64)


def _block(x, pos, nfram, ln, per, fill_k):
    """the block's rows, with the frames at or after each unit's length overwritten with a non-finite or huge value"""
    blk = np.array(x[:, pos:pos + nfram])
    for u, L in enumerate(ln):
        blk[u * per:(u + 1) * per, L:] = FILL[(fill_k + u) % len(FILL)]
    return blk


def _feed(blk, host):
    import torch
    return blk if host else torch.from_numpy(blk).cuda()


# ---------------------------------------------------------------------------------------------------------------- true peak / K-meter
class _TpkPriv:
    def __init__(self, n, flags, fsamp=48000.0):
        self.flags = flags
        self.tp = [O.TruePeak(1, fsamp) for _ in range(n)] if flags & 1 else None
        self.km = [O.Kmeter(1, fsamp) for _ in range(n)] if flags & 2 else None
        self.want = np.zeros((n, 4), np.float32)        # tp_m tp_p km_rms km_peak as last read

    def feed(self, blk, ln, read=True):
        for i, L in enumerate(ln):
            if L == 0:
                continue
            xi = np.ascontiguousarray(blk[i:i + 1, :L])
            if self.tp:
                self.tp[i].process(xi)
                if read:
                    m, p = self.tp[i].read(); self.want[i, 0], self.want[i, 1] = m[0], p[0]
            if self.km:
                self.km[i].process(xi)
                if read:
                    r, p = self.km[i].read(); self.want[i, 2], self.want[i, 3] = r[0], p[0]

    def state(self, rows):
        out = {}
        if self.tp:
            pk = [self.tp[i].peek() for i in rows]
            for k, name in enumerate(("m", "p", "z1", "z2")):
                out[name] = np.array([q[k][0] for q in pk], np.float32)
            out["res"] = np.array([q[4][0] for q in pk], np.int32)
        if self.km:
            out["km"] = np.concatenate([self.km[i].peek() for i in rows])
        return out


def _tpk_check(tag, g, priv, rows, fma=False):
    r = g.read()
    got = np.stack([r["tp_m"], r["tp_p"], r["km_rms"], r["km_peak"]], 1)[rows]
    want = priv.want[rows]
    cols = ([0, 1] if priv.flags & 1 else []) + ([2, 3] if priv.flags & 2 else [])
    for c in cols:
        if fma:                                             # tolerance mode: the fused FIR and the contracted K-meter filters
            live = want[:, c] > 1e-10
            assert np.array_equal(live, got[:, c] > 1e-10), (tag, c)
            assert np.abs(_db(got[live, c]) - _db(want[live, c])).max(initial=0) <= 1e-4, (tag, c)
        else:
            assert np.array_equal(u32(got[:, c]), u32(want[:, c])), (tag, c, np.nonzero(u32(got[:, c]) != u32(want[:, c]))[0][:5])


def _tpk_state_check(tag, g, priv, rows):
    s = g.state(); w = priv.state(rows)
    for k, v in w.items():
        a = s[k][rows]
        assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a, v.view(np.uint32) if v.dtype == np.float32 else v), (tag, k)


@pytest.mark.parametrize("flags", [3, 1, 2])
@pytest.mark.parametrize("host", [False, True])
def test_tpk_ragged_bit_exact(flags, host):
    import meters_lv2_b200 as B
    n = 40
    rng = np.random.default_rng(100 + flags)
    x = _signal(n, sum(SIZES), seed=flags)
    g = B.TruePeakKmeter(n, flags=flags)
    priv = _TpkPriv(n, flags)
    rows = np.arange(n)
    pos = 0
    for b, nfram in enumerate(SIZES):
        ln = _lengths(rng, n, nfram, b, sit_out=[2, 17, 33])
        blk = _block(x, pos, nfram, ln, 1, b)
        g.process(_feed(blk, host), lengths=ln)
        priv.feed(blk, ln)
        _tpk_check(("tpk", flags, host, b), g, priv, rows)
        pos += nfram
    _tpk_state_check(("tpk", flags, host), g, priv, rows)


@pytest.mark.parametrize("flags", [3, 1])
def test_tpk_ragged_in_tolerance_mode(flags):
    """a B200M_PREC_FMA bank: ragged blocks run the exact kernel, plain ones the tolerance-mode kernels; readings within +-1e-4 dB"""
    import meters_lv2_b200 as B
    n = 24
    rng = np.random.default_rng(7)
    x = _signal(n, sum(SIZES), seed=9)
    g = B.TruePeakKmeter(n, flags=flags); g.set_precision(B.PREC_FMA)
    priv = _TpkPriv(n, flags)
    pos = 0
    for b, nfram in enumerate(SIZES):
        ln = _lengths(rng, n, nfram, b, sit_out=[5]) if b % 3 else np.full(n, nfram)
        blk = _block(x, pos, nfram, ln, 1, b)
        g.process(_feed(blk, False), lengths=None if b % 3 == 0 else ln)
        priv.feed(blk, ln)
        _tpk_check(("tpk fma", b), g, priv, np.arange(n), fma=True)
        pos += nfram


def test_tpk_snapshot_after_ragged_block_restores_and_continues():
    import meters_lv2_b200 as B
    L = B.lib()
    n, nfram = 20, 1024
    rng = np.random.default_rng(11)
    x = _signal(n, 6 * nfram, seed=12)
    a = B.TruePeakKmeter(n)
    for b in range(3):
        ln = _lengths(rng, n, nfram, b, sit_out=[])
        a.process(_feed(_block(x, b * nfram, nfram, ln, 1, b), False), lengths=ln)
    a.read()
    size = L.b200m_tpk_snapshot_size(a.h)
    buf = (C.c_uint8 * size)()
    B._ck(L.b200m_tpk_snapshot(a.h, buf, size, B._stream_ptr(None)))
    c = B.TruePeakKmeter(n)
    B._ck(L.b200m_tpk_restore(c.h, buf, size, B._stream_ptr(None)))
    for b in range(3, 6):
        ln = _lengths(rng, n, nfram, b, sit_out=[4])
        blk = _feed(_block(x, b * nfram, nfram, ln, 1, b), False)
        a.process(blk, lengths=ln); c.process(blk, lengths=ln)
        ra, rc = a.read(), c.read()
        assert ra.tobytes() == rc.tobytes(), b
    sa, sc = a.state(), c.state()
    for k in sa:
        assert sa[k].tobytes() == sc[k].tobytes(), k


# ---------------------------------------------------------------------------------------------------------------- needle meters
class _PpmPriv:
    def __init__(self, n, kind):
        self.kind, self.per = kind, 2 if kind == O.PPM_MS else 1
        self.o = [O.Needle(1, kind) for _ in range(n)]
        self.want = np.zeros(n * self.per, np.float32)

    def feed(self, blk, ln):
        for u, L in enumerate(ln):
            if L == 0:
                continue
            self.o[u].process(np.ascontiguousarray(blk[u * self.per:(u + 1) * self.per, :L]))
            self.want[u * self.per:(u + 1) * self.per] = self.o[u].read()

    def state(self, units):
        return np.concatenate([self.o[u].peek() for u in units])


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
@pytest.mark.parametrize("host", [False, True])
def test_ppm_ragged_bit_exact(kind, host):
    import meters_lv2_b200 as B
    n = 40
    rng = np.random.default_rng(200 + kind)
    priv = _PpmPriv(n, kind)
    x = _signal(n * priv.per, sum(SIZES), seed=20 + kind)
    g = B.NeedleMeters(n, kind)
    pos = 0
    for b, nfram in enumerate(SIZES):
        ln = _lengths(rng, n, nfram, b, sit_out=[1, 9, 30])
        if kind == B.PPM_MS and b in (2, 4, 8):
            # M/S gains, also on pairs that sit out the next blocks: they apply from the pair's next call, as on a private meter
            for u in (1, 9, 12) if b < 8 else (30,):
                dm, ds = float(rng.uniform(-20, 6)), float(rng.uniform(-20, 6))
                g.set_gain(dm, ds, unit=u); priv.o[u].set_gain(dm, ds)
        blk = _block(x, pos, nfram, ln, priv.per, b)
        g.process(_feed(blk, host), lengths=ln)
        priv.feed(blk, ln)
        got = g.read()
        assert np.array_equal(u32(got), u32(priv.want)), (kind, host, b, np.nonzero(u32(got) != u32(priv.want))[0][:5])
        pos += nfram
    assert np.array_equal(u32(g.state()), u32(priv.state(range(n))))


# ---------------------------------------------------------------------------------------------------------------- correlation
class _CorPriv:
    def __init__(self, n):
        self.o = [O.Stcorr(1) for _ in range(n)]

    def feed(self, blk, ln):
        for i, L in enumerate(ln):
            if L:
                self.o[i].process(np.ascontiguousarray(blk[2 * i:2 * i + 2, :L]))

    def read(self, idx):
        return np.array([self.o[i].read()[0] for i in idx], np.float32)

    def state(self, idx):
        return np.concatenate([self.o[i].peek() for i in idx])


@pytest.mark.parametrize("scan", [False, True])
@pytest.mark.parametrize("host", [False, True])
def test_cor_ragged(scan, host):
    import meters_lv2_b200 as B
    n = 40
    rng = np.random.default_rng(300 + scan)
    x = _signal(2 * n, sum(SIZES), seed=30)
    x[1::2] = 0.6 * x[0::2] + 0.4 * x[1::2]                 # correlated pairs
    g = B.Stcorrdsp(n)
    if scan:
        g.set_precision(B.PREC_FMA)
    priv = _CorPriv(n)
    pos = 0
    for b, nfram in enumerate(SIZES):
        ln = _lengths(rng, n, nfram, b, sit_out=[0, 21, 39])
        blk = _block(x, pos, nfram, ln, 2, b)
        g.process(_feed(blk, host), lengths=ln)
        priv.feed(blk, ln)
        got, want = g.read(), priv.read(range(n))
        if scan:
            assert np.abs(got.astype(np.float64) - want).max() <= 1e-5, (b, np.abs(got - want).max())
        else:
            assert np.array_equal(u32(got), u32(want)), (b, np.nonzero(u32(got) != u32(want))[0][:5])
            assert np.array_equal(u32(g.state()), u32(priv.state(range(n)))), b
        pos += nfram


def test_cor_ragged_refused_while_attached_to_a_phasewheel():
    import torch
    import meters_lv2_b200 as B
    n = 8
    cor = B.Stcorrdsp(n); pw = B.Phasewheel(n)
    pw.attach_cor(cor)
    x = torch.zeros(2 * n, 256, device="cuda")
    ln = np.full(n, 100)
    n0 = B.launch_count()
    with pytest.raises(B.B200MError, match="attached to a phasewheel"):
        cor.process(x, lengths=ln)
    assert B.launch_count() == n0
    cor.process(x, run=np.ones(n, np.uint8))                # the hold keeps working on an attached bank
    pw.attach_cor(None)
    cor.process(x, lengths=ln)


# ---------------------------------------------------------------------------------------------------------------- spectrum
class _SpecPriv:
    def __init__(self, n, nchan):
        self.nchan = nchan
        self.o = [O.Spectr30(1, nchan) for _ in range(n)]
        self.want = np.zeros((n, 60), np.float32)

    def feed(self, blk, ln, spd, rst):
        c = self.nchan
        for i, L in enumerate(ln):
            if L:
                self.o[i].process(np.ascontiguousarray(blk[c * i:c * (i + 1), :L]), float(spd[i]), float(rst[i]))
                self.want[i] = self.o[i].read()[0]


def _spec_check(tag, got, want, fma):
    pending = want[:, 30:] <= -500                           # reset handshake cycles: the reference emits -500 - rand()
    assert np.array_equal(pending, got[:, 30:] <= -500), tag
    g = np.concatenate([got[:, :30].ravel(), got[:, 30:][~pending]])
    w = np.concatenate([want[:, :30].ravel(), want[:, 30:][~pending]])
    if fma:
        live = w > -100
        assert np.array_equal(live, g > -100), tag
        assert np.abs(g[live].astype(np.float64) - w[live]).max(initial=0) <= 1e-4, tag
    else:
        assert np.array_equal(u32(g), u32(w)), (tag, np.abs(g - w).max())


@pytest.mark.parametrize("nchan,fma,host", [(2, False, False), (1, False, True), (2, True, False), (2, False, True)])
def test_spec_ragged_with_instance_controls(nchan, fma, host):
    import meters_lv2_b200 as B
    n = 12
    rng = np.random.default_rng(400 + nchan + 2 * fma)
    sizes = SIZES[:9]
    x = _signal(nchan * n, sum(sizes), seed=40)
    g = B.Spectr30(n, nchan)
    if fma:
        g.set_precision(B.PREC_FMA)
    priv = _SpecPriv(n, nchan)
    pos = 0
    for b, nfram in enumerate(sizes):
        ln = _lengths(rng, n, nfram, b, sit_out=[3, 7])
        # per-instance speed and reset ports, changing on instances that run and on ones that sit out (their rows are ignored)
        spd = np.where(np.arange(n) % 3 == 0, 1.0 + (b // 2), 5.0).astype(np.float32)
        rst = np.full(n, -4.0, np.float32)
        rst[(np.arange(n) + b) % 4 == 0] = float((b % 3) + 1)
        rst[7] = 1.0 if b in (4, 5) else -4.0               # a handshake started while instance 7 sits out: it must not advance
        blk = _block(x, pos, nfram, ln, nchan, b)
        g.process(_feed(blk, host), speed=spd, reset=rst, lengths=ln)
        priv.feed(blk, ln, spd, rst)
        _spec_check((nchan, fma, host, b), g.read(), priv.want, fma)
        pos += nfram
    if not fma:
        for i in (0, 3, n - 1):
            z, v, m = g.state(i); oz, ov, om = priv.o[i].state(0)
            assert np.array_equal(z.view(np.uint64), oz.view(np.uint64)) and np.array_equal(u32(v), u32(ov)) and np.array_equal(u32(m), u32(om)), i


# ---------------------------------------------------------------------------------------------------------------- every bank
def _banks(B, kind):
    """(make a bank, rows per unit, units, process(bank, x, lengths), read(bank))"""
    if kind == "tpk":
        return (lambda: B.TruePeakKmeter(48), 1, 48, lambda g, x, ln, **k: g.process(x, lengths=ln, **k), lambda g: g.read().tobytes() + g.state()["km"].tobytes())
    if kind == "tp":
        return (lambda: B.TruePeakKmeter(48, flags=1), 1, 48, lambda g, x, ln, **k: g.process(x, lengths=ln, **k), lambda g: g.read().tobytes() + g.state()["z1"].tobytes())
    if kind == "ppm":
        return (lambda: B.NeedleMeters(40, B.PPM_MS), 2, 40, lambda g, x, ln, **k: g.process(x, lengths=ln, **k), lambda g: g.read().tobytes() + g.state().tobytes())
    if kind == "vu":
        return (lambda: B.NeedleMeters(40, B.PPM_VU), 1, 40, lambda g, x, ln, **k: g.process(x, lengths=ln, **k), lambda g: g.read().tobytes() + g.state().tobytes())
    if kind == "cor":
        return (lambda: B.Stcorrdsp(40), 2, 40, lambda g, x, ln, **k: g.process(x, lengths=ln, **k), lambda g: g.read().tobytes() + g.state().tobytes())
    if kind == "spec":
        def proc(g, x, ln, **k):
            g.process(x, speed=np.full(12, 2.0, np.float32), reset=np.full(12, -4.0, np.float32), lengths=ln, **k)
        return (lambda: B.Spectr30(12, 2), 2, 12, proc, lambda g: g.read().tobytes() + g.state(5)[0].tobytes())
    raise ValueError(kind)


KINDS = ["tpk", "tp", "ppm", "vu", "cor", "spec"]


@pytest.mark.parametrize("kind", KINDS)
def test_uniform_lengths_are_the_plain_call(kind):
    """every length nfram: the same bits and the same launches as the plain call (on twin banks)"""
    import torch
    import meters_lv2_b200 as B
    make, per, n, proc, rd = _banks(B, kind)
    a, c = make(), make()
    x = torch.from_numpy(_signal(per * n, 3 * 1024, seed=5)).cuda()
    for b in range(3):
        xb = x[:, b * 1024:(b + 1) * 1024]
        torch.cuda.synchronize()
        n0 = B.launch_count(); proc(a, xb, None); n1 = B.launch_count(); proc(c, xb, np.full(n, 1024)); n2 = B.launch_count()
        assert n1 - n0 == n2 - n1, (kind, b)
        assert rd(a) == rd(c), (kind, b)


@pytest.mark.parametrize("kind", KINDS)
def test_length_above_nfram_is_refused(kind):
    import torch
    import meters_lv2_b200 as B
    make, per, n, proc, rd = _banks(B, kind)
    g = make()
    x = torch.from_numpy(_signal(per * n, 1024, seed=6)).cuda()
    proc(g, x, np.arange(n) % 1024)
    before = rd(g)
    ln = np.full(n, 512); ln[n // 2] = 1025
    torch.cuda.synchronize()
    n0 = B.launch_count()
    with pytest.raises(B.B200MError, match="exceeds nfram"):
        proc(g, x, ln)
    assert B.launch_count() == n0
    assert rd(g) == before


@pytest.mark.parametrize("kind", KINDS)
def test_path_switches_and_a_caller_stream_between_ragged_blocks(kind):
    """schedule D H D D H H D on a busy caller stream against a twin bank driven on the device path only"""
    import torch
    import meters_lv2_b200 as B
    make, per, n, proc, rd = _banks(B, kind)
    a, c = make(), make()
    rng = np.random.default_rng(77)
    side = torch.cuda.Stream()
    pos = 0
    x = _signal(per * n, 7 * 4097, seed=8)
    for b, path in enumerate("DHDDHHD"):
        nfram = (1024, 4097, 333, 4097, 1024, 64, 2000)[b]
        ln = _lengths(rng, n, nfram, b, sit_out=[1])
        blk = _block(x, pos, nfram, ln, per, b)
        pos += nfram
        if path == "H":
            proc(a, blk, ln)
        else:
            with torch.cuda.stream(side):
                torch.cuda._sleep(2_000_000)
                xd = torch.from_numpy(blk).to("cuda", non_blocking=False)
                proc(a, xd, ln, stream=side)
        proc(c, torch.from_numpy(blk).cuda(), ln)
    side.synchronize(); torch.cuda.synchronize()
    assert rd(a) == rd(c), kind


# ---------------------------------------------------------------------------------------------------------------- bank sizes of the cost script
def _sample(n, k, seed):
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([[0, n - 1], rng.choice(n, k, replace=False)]))


@pytest.mark.parametrize("kind", ["tpk", "vu", "iec2", "cor", "cor_scan", "spec", "spec_fma"])
def test_ragged_at_full_size_against_sampled_private_instances(kind):
    import torch
    import meters_lv2_b200 as B
    nfram, nblk = 1024, 3
    units = {"tpk": 16384, "vu": 16384, "iec2": 16384, "cor": 8192, "cor_scan": 8192, "spec": 4096, "spec_fma": 4096}[kind]
    per = {"tpk": 1, "vu": 1, "iec2": 1}.get(kind, 2)
    sel = _sample(units, 30, 1)
    rng = np.random.default_rng(5)
    if kind == "tpk":
        g = B.TruePeakKmeter(units); priv = _TpkPriv(len(sel), 3)
    elif kind in ("vu", "iec2"):
        g = B.NeedleMeters(units, B.PPM_VU if kind == "vu" else B.PPM_IEC2); priv = _PpmPriv(len(sel), B.PPM_VU if kind == "vu" else B.PPM_IEC2)
    elif kind.startswith("cor"):
        g = B.Stcorrdsp(units); priv = _CorPriv(len(sel))
        if kind == "cor_scan":
            g.set_precision(B.PREC_FMA)
    else:
        g = B.Spectr30(units, 2); priv = _SpecPriv(len(sel), 2)
        if kind == "spec_fma":
            g.set_precision(B.PREC_FMA)
    gen = torch.Generator(device="cuda").manual_seed(3)
    for b in range(nblk):
        ln = _lengths(rng, units, nfram, b + 3, sit_out=sel[::4])
        xd = (torch.rand(per * units, nfram, device="cuda", generator=gen) - 0.5) * 0.8
        cols = torch.arange(nfram, device="cuda")[None, :]
        lt = torch.from_numpy(np.repeat(ln, per)).cuda()[:, None]
        xd = torch.where(cols >= lt, torch.full_like(xd, float("nan")), xd).contiguous()
        rows = np.concatenate([np.arange(u * per, (u + 1) * per) for u in sel])
        blk = xd[torch.from_numpy(rows).cuda()].cpu().numpy()
        lsel = ln[sel]
        if kind.startswith("spec"):
            g.process(xd, speed=1.0, reset=-4.0, lengths=ln)
            priv.feed(blk, lsel, np.ones(len(sel)), np.full(len(sel), -4.0))
            _spec_check((kind, b), g.read()[sel], priv.want, kind == "spec_fma")
        elif kind == "tpk":
            g.process(xd, lengths=ln); priv.feed(blk, lsel)
            r = g.read()
            got = np.stack([r["tp_m"], r["tp_p"], r["km_rms"], r["km_peak"]], 1)[sel]
            assert np.array_equal(u32(got), u32(priv.want)), (kind, b)
        elif kind in ("vu", "iec2"):
            g.process(xd, lengths=ln); priv.feed(blk, lsel)
            assert np.array_equal(u32(g.read()[sel]), u32(priv.want)), (kind, b)
        else:
            g.process(xd, lengths=ln); priv.feed(blk, lsel)
            got, want = g.read()[sel], priv.read(range(len(sel)))
            if kind == "cor_scan":
                assert np.abs(got.astype(np.float64) - want).max() <= 1e-5, (kind, b)
            else:
                assert np.array_equal(u32(got), u32(want)), (kind, b)
