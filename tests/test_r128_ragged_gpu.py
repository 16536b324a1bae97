"""GPU: ragged blocks of the EBU R128 and EBUr128 banks (b200m_ebu_process_ragged_*, b200m_r128_run_ragged_*) and
programme_loudness.

Every bank instance i is compared with a private reference instance that sees only its own frames: one Ebu_r128_proc (the
reference build, or for weighted layouts the restatement in tests/_ebu_weighted.cc) and one TruePeakdsp set per instance, fed the
first len[i] frames of each block with len[i] > 0, with the dBTP fold of src/ebulv2.cc:360-367.  Frames at or after len[i] hold NaN.
"""
import ctypes as C

import numpy as np
import pytest

import _ebu_weighted as W
import _oracle as O

pytestmark = pytest.mark.gpu
RES = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")
_libm = C.CDLL("libm.so.6")
_libm.log10f.restype = C.c_float
_libm.log10f.argtypes = [C.c_float]


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _db(v):
    """coef_to_db (src/ebulv2.cc:227-230)"""
    return np.float32(-np.inf) if v == 0 else np.float32(20.0 * float(_libm.log10f(float(v))))


def _gains(layout):
    import meters_lv2_b200 as B
    if layout == "7.1.4":
        return B.bs1770_weights([30, -30, 0, 90, -90, 135, -135, 45, -45, 135, -135], [0] * 7 + [35] * 4)
    if layout == "5.1":
        return np.float32([1, 1, 1, 0, 1.41, 1.41])
    return None


class _Priv:
    """a private reference instance: Ebu_r128_proc + nchan TruePeakdsp + the EBUr128 dBTP hold"""

    def __init__(self, nchan, gains, fs):
        self.nc, self.g, self.fs = nchan, gains, fs
        self.ebu = O.Ebu(1, nchan, fs) if gains is None else W.Ebu(1, gains, fs)
        self.fresh_tp()
        self.on = True

    def fresh_tp(self):
        self.tp = O.TruePeak(self.nc, self.fs)
        self.hold = np.float32(-np.inf)

    def new(self):
        """B200M_R128_NEW: a freshly instantiated plugin"""
        self.ebu = O.Ebu(1, self.nc, self.fs) if self.g is None else W.Ebu(1, self.g, self.fs)
        self.fresh_tp()

    def run(self, xi, dbtp=True):
        """one plugin cycle over xi [nchan, L], L > 0"""
        self.ebu.process(xi)
        if not dbtp:
            return
        if not self.on:
            self.hold = np.float32(-np.inf)
            return
        self.tp.process(xi, mode=1)
        m, _ = self.tp.read()
        t = m[0]
        for c in range(1, self.nc):
            t = t if t > m[c] else m[c]
        tp = _db(t)
        if tp > self.hold:
            self.hold = tp


def _feed(privs, x, lens, dbtp=True):
    for i, p in enumerate(privs):
        if lens[i]:
            p.run(np.ascontiguousarray(x[i * p.nc:(i + 1) * p.nc, :lens[i]]), dbtp)


def _check(tag, bank, privs, ok=None, tol=False, state=True):
    """every loudness float, frag_power, both histograms and counts, the instance state and the hold, per instance"""
    r, tp = bank.results()
    for i, p in enumerate(privs):
        if ok is not None and not ok[i]:
            continue
        want = p.ebu.read()[0]
        for k, name in enumerate(RES):
            assert u32(r[name][i]) == u32(want[k]), (tag, i, name, r[name][i], want[k])
        hm, hs = bank.ebu.histogram(i)
        om, os_, oc = p.ebu.hist(0)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_), (tag, i)
        assert r["hist_M_count"][i] == oc[0] and r["hist_S_count"][i] == oc[1], (tag, i)
        if state and p.g is None:
            z, pw, fr, c = bank.ebu.state(i)
            oz, opw, ofr, oc4 = p.ebu.state(0)
            assert np.array_equal(u32(z), u32(oz)), (tag, i, "z")
            assert np.array_equal(u32(pw), u32(opw)), (tag, i, "ring")
            assert u32(fr) == u32(ofr), (tag, i, "frpwr")
            assert np.array_equal(np.asarray(c), np.asarray(oc4)), (tag, i, "counters", c, oc4)
            assert u32(r["frag_power"][i]) == u32(opw[(oc4[1] - 1) % 64]), (tag, i, "frag_power")
    want = np.float32([p.hold for p in privs])
    if tol:
        fin = np.isfinite(want)
        assert np.array_equal(np.isfinite(tp), fin) and np.array_equal(tp[~fin], want[~fin]), tag
        assert np.all(np.abs(tp[fin].astype(np.float64) - want[fin]) <= 1e-4), (tag, np.max(np.abs(tp[fin] - want[fin])))
    else:
        assert np.array_equal(u32(tp), u32(want)), (tag, np.nonzero(u32(tp) != u32(want))[0][:5])


def _snapshot(bk):
    """the bank's snapshot written into a zeroed buffer (the blob's alignment padding is never written)"""
    import meters_lv2_b200 as B
    n = B.lib().b200m_r128_snapshot_size(bk.h)
    buf = np.zeros(n, np.uint8)
    B._ck(B.lib().b200m_r128_snapshot(bk.h, B._np_ptr(buf), n, None))
    return buf


def _signal(rng, rows, n):
    lvl = 10.0 ** rng.uniform(-3.0, 0.0, size=(rows, 1))
    lvl[::13] = 0.0
    x = rng.standard_normal((rows, n)).astype(np.float32) * 0.3
    x += 0.5 * np.sin(2 * np.pi * rng.uniform(40, 4000, size=(rows, 1)) * np.arange(n) / 48000.0).astype(np.float32)
    return (x * lvl).astype(np.float32)


def _lengths(rng, privs, nfram):
    """per instance one of {0, 1, 3, 4, 47, 48, 49, own next fragment edge -1 / 0 / +1, nfram}, clamped to nfram"""
    out = np.empty(len(privs), np.uint32)
    for i, p in enumerate(privs):
        cand = [0, 1, 3, 4, 47, 48, 49, nfram, nfram]
        if p.g is None:
            e = int(p.ebu.state(0)[3][0])
            cand += [e - 1, e, e + 1]
        else:
            cand += [1199, 1200, 1201]
        out[i] = min(max(int(cand[int(rng.integers(len(cand)))]), 0), nfram)
    return out


NFRAMS = [1024, 1024, 1000, 2400, 4097, 64, 7, 8192]


@pytest.mark.parametrize("layout,nchan,fs,n_inst,path,prec", [
    ("mono", 1, 48000.0, 37, "device", 0),
    ("stereo", 2, 48000.0, 41, "device", 0),
    ("stereo", 2, 44100.0, 23, "device", 1),
    ("5ch", 5, 44100.0, 29, "device", 0),
    ("7.1.4", 11, 48000.0, 21, "device", 0),
    ("stereo", 2, 48000.0, 64, "host1", 0),
    ("5ch", 5, 48000.0, 64, "host4", 1),
    ("7.1.4", 11, 44100.0, 64, "host8", 0),
])
def test_ragged_parity_every_block(layout, nchan, fs, n_inst, path, prec, monkeypatch):
    """200 blocks of random per-instance lengths, NaN past each end: every field bit-identical to private instances after every
    block (tolerance mode: the hold within 1e-4 dB, everything else bitwise)"""
    import torch
    import meters_lv2_b200 as B
    if path.startswith("host"):
        monkeypatch.setenv("B200M_R128_SLICES", path[4:])
    g = _gains(layout)
    bank = B.EBUr128(n_inst, fs, True, nchan=nchan, gains=g)
    bank.set_precision(prec)
    bank.control(B.EBUr128.START)
    privs = [_Priv(nchan, g, fs) for _ in range(n_inst)]
    for p in privs:
        p.ebu.integr("start")
    rng = np.random.default_rng(nchan * 100 + n_inst + int(fs))
    for b in range(200):
        nfram = NFRAMS[int(rng.integers(len(NFRAMS)))]
        x = _signal(rng, n_inst * nchan, nfram)
        lens = _lengths(rng, privs, nfram)
        if b % 17 == 0:
            lens[:] = nfram                                  # a uniform block in between: the plain call
        xs = x.copy()
        for i in range(n_inst):
            xs[i * nchan:(i + 1) * nchan, lens[i]:] = np.nan
        if path == "device":
            bank.run(torch.from_numpy(xs).cuda(), lengths=lens)
        else:
            bank.run(xs, lengths=lens)
        _feed(privs, x, lens)
        _check((layout, path, b), bank, privs, tol=prec == 1)


@pytest.mark.parametrize("nchan,layout,n_inst,prec", [(1, None, 37, 0), (2, None, 41, 1), (5, None, 29, 0), (11, "7.1.4", 13, 1),
                                                      (2, None, 5120, 1)])
def test_uniform_lengths_are_the_plain_call(nchan, layout, n_inst, prec):
    """every length = nfram: the plain call's bits and launch count, device and host path (5120 stereo instances: the fused kernel)"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _gains(layout)
    rng = np.random.default_rng(n_inst)
    for host in (False, True):
        a, b = E(n_inst, 48000.0, True, nchan=nchan, gains=g), E(n_inst, 48000.0, True, nchan=nchan, gains=g)
        for bk in (a, b):
            bk.set_precision(prec); bk.control(E.START)
        for k in range(6):
            nfram = (1024, 1000, 4096)[k % 3]
            xh = _signal(rng, n_inst * nchan, nfram)
            x = xh if host else torch.from_numpy(xh).cuda()
            full = np.full(n_inst, nfram, np.uint32)
            torch.cuda.synchronize()
            l0 = B.launch_count(); a.run(x); torch.cuda.synchronize(); la = B.launch_count() - l0
            l0 = B.launch_count(); b.run(x, lengths=full); torch.cuda.synchronize(); lb = B.launch_count() - l0
            assert la == lb, (host, k, la, lb)
            ra, ta = a.results(); rb, tb = b.results()
            assert ra.tobytes() == rb.tobytes() and u32(ta).tobytes() == u32(tb).tobytes(), (host, k)
        for i in (0, n_inst - 1):
            assert all(np.array_equal(p, q) for p, q in zip(a.histogram(i), b.histogram(i)))
        assert _snapshot(a).tobytes() == _snapshot(b).tobytes()
        a.close(); b.close()


@pytest.mark.parametrize("nchan,layout", [(2, None), (5, None), (6, "5.1")])
def test_controls_dbtp_and_checkpoint(nchan, layout):
    """START / PAUSE / RESET / NEW / CLEAR and per-instance dBTP between ragged blocks, a snapshot after ragged blocks restored into
    a fresh bank: both banks continue bit-identical to each other and to the private instances"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    fs, n_inst = 48000.0, 31
    g = _gains(layout)
    bank = E(n_inst, fs, True, nchan=nchan, gains=g)
    bank.control(E.START)
    privs = [_Priv(nchan, g, fs) for _ in range(n_inst)]
    for p in privs:
        p.ebu.integr("start")
    ok = np.ones(n_inst, bool)                 # CLEAR keeps the fragment clock: no private counterpart of its EBU part until a NEW
    rng = np.random.default_rng(nchan)
    banks = [bank]
    for b in range(160):
        if b >= 2 and b % 2 == 0:
            for _ in range(2):
                i = int(rng.integers(n_inst))
                cmd = ("start", "pause", "reset", "clear", "new", "dbtp", "dbtp")[int(rng.integers(7))]
                for bk in banks:
                    if cmd == "dbtp":
                        bk.set_dbtp(not privs[i].on, i)
                    else:
                        bk.control({"start": E.START, "pause": E.PAUSE, "reset": E.RESET, "clear": E.CLEAR, "new": E.NEW}[cmd], i)
                p = privs[i]
                if cmd == "dbtp":
                    p.on = not p.on
                elif cmd in ("start", "pause"):
                    p.ebu.integr(cmd)
                elif cmd == "reset":
                    p.ebu.integr("reset"); p.hold = np.float32(-np.inf)
                elif cmd == "clear":
                    ok[i] = False; p.fresh_tp()
                else:
                    p.new(); ok[i] = True
        if b == 80:                            # checkpoint: a fresh bank restored from the snapshot runs alongside
            twin = E(n_inst, fs, True, nchan=nchan, gains=g)
            twin.restore(bank.snapshot())
            banks.append(twin)
        nfram = NFRAMS[int(rng.integers(len(NFRAMS)))]
        x = _signal(rng, n_inst * nchan, nfram)
        lens = _lengths(rng, privs, nfram)
        xs = x.copy()
        for i in range(n_inst):
            xs[i * nchan:(i + 1) * nchan, lens[i]:] = np.nan
        xd = torch.from_numpy(xs).cuda()
        for bk in banks:
            bk.run(xd if bk is bank else xs, lengths=lens)
        _feed(privs, x, lens)
        for bk in banks:
            _check((nchan, b), bk, privs, ok=ok)
        if len(banks) == 2:
            ra, ta = banks[0].results(); rb, tb = banks[1].results()
            assert ra.tobytes() == rb.tobytes() and u32(ta).tobytes() == u32(tb).tobytes(), b
    assert _snapshot(banks[0]).tobytes() == _snapshot(banks[1]).tobytes()


def test_ebu_bank_ragged_and_invalid_lengths():
    """the EBU bank alone: ragged device and host calls against private instances; a length > nfram is B200M_E_INVAL and changes
    nothing (snapshot, launch count); len = NULL is the plain call"""
    import torch
    import meters_lv2_b200 as B
    L = B.lib()
    n_inst, nchan, fs = 19, 2, 48000.0
    a, b = B.Ebu_r128_proc(n_inst, nchan, fs), B.Ebu_r128_proc(n_inst, nchan, fs)
    privs = [O.Ebu(1, nchan, fs) for _ in range(n_inst)]
    for e in (a, b):
        e.integr_start()
    for p in privs:
        p.integr("start")
    rng = np.random.default_rng(5)
    for k in range(120):
        nfram = NFRAMS[k % len(NFRAMS)]
        x = _signal(rng, n_inst * nchan, nfram)
        lens = rng.choice([0, 1, 47, 48, 49, 2399, 2400, 2401, nfram], size=n_inst).clip(0, nfram).astype(np.uint32)
        xs = x.copy()
        for i in range(n_inst):
            xs[i * nchan:(i + 1) * nchan, lens[i]:] = np.nan
        a.process(torch.from_numpy(xs).cuda(), lengths=lens)
        b.process(xs, lengths=lens)
        torch.cuda.synchronize()
        for i, p in enumerate(privs):
            if lens[i]:
                p.process(np.ascontiguousarray(x[i * nchan:(i + 1) * nchan, :lens[i]]))
        want = np.stack([p.read()[0] for p in privs])
        for e in (a, b):
            r = e.results()
            for j, name in enumerate(RES):
                assert np.array_equal(u32(r[name]), u32(want[:, j])), (k, name)
        for i in (0, 7, n_inst - 1):
            for e in (a, b):
                z, pw, fr, c = e.state(i); oz, opw, ofr, oc = privs[i].state(0)
                assert np.array_equal(u32(z), u32(oz)) and np.array_equal(u32(pw), u32(opw)) and np.array_equal(c, oc), (k, i)
    # invalid: one length above nfram
    x = torch.zeros(n_inst * nchan, 256, device="cuda")
    bad = np.full(n_inst, 256, np.uint32); bad[3] = 257
    n = L.b200m_ebu_snapshot_size(a.h)
    s0 = np.zeros(n, np.uint8); B._ck(L.b200m_ebu_snapshot(a.h, B._np_ptr(s0), n, None))
    torch.cuda.synchronize()
    l0 = B.launch_count()
    assert L.b200m_ebu_process_ragged_device(a.h, C.c_void_p(x.data_ptr()), 256, 256, B._np_ptr(bad), None) == -1
    hx = np.zeros((n_inst * nchan, 256), np.float32)
    assert L.b200m_ebu_process_ragged_host(b.h, B._np_ptr(hx), 256, 256, B._np_ptr(bad)) == -1
    assert B.launch_count() == l0
    s1 = np.zeros(n, np.uint8); B._ck(L.b200m_ebu_snapshot(a.h, B._np_ptr(s1), n, None))
    assert s0.tobytes() == s1.tobytes()
    # NULL lengths: the plain call
    r128 = [B.EBUr128(n_inst, fs, True), B.EBUr128(n_inst, fs, True)]
    xr = torch.from_numpy(_signal(rng, n_inst * 2, 1024)).cuda()
    B._ck(L.b200m_r128_run_ragged_device(r128[0].h, C.c_void_p(xr.data_ptr()), 1024, 1024, None, None))
    r128[1].run(xr)
    bad = np.full(n_inst, 1024, np.uint32); bad[0] = 1025
    assert L.b200m_r128_run_ragged_device(r128[0].h, C.c_void_p(xr.data_ptr()), 1024, 1024, B._np_ptr(bad), None) == -1
    (ra, ta), (rb, tb) = r128[0].results(), r128[1].results()
    assert ra.tobytes() == rb.tobytes() and u32(ta).tobytes() == u32(tb).tobytes()


# ---- programme_loudness ----------------------------------------------------------------------------------------------------
def _clip(seed, i, off, n, nchan, fs):
    """frames off .. off + n - 1 of clip i: a level, a slow swell, a tone per channel and noise drawn from (seed, clip, offset)"""
    rng = np.random.default_rng((seed, i, off))
    t = (off + np.arange(1024)) / fs                         # always a whole 1024-frame block, cut to n: the same frames for any n
    c = np.arange(nchan)[:, None]
    lvl = 10.0 ** (-2.5 * ((i * 0.37) % 1.0))
    swell = 0.6 + 0.4 * np.sin(2 * np.pi * (0.05 + 0.01 * (i % 7)) * t)
    x = rng.standard_normal((nchan, 1024)) * 0.25 + 0.3 * np.sin(2 * np.pi * (110.0 + 17.0 * (c + i)) * t)
    return np.ascontiguousarray((x * lvl * swell).astype(np.float32)[:, :n])


def _private_programme(get, i, length, nchan, gains, fs, block):
    """clip i (get (off, n): its frames) through a private instance in blocks of `block` frames with a short last block"""
    p = _Priv(nchan, gains, fs)
    p.ebu.integr("start")
    for off in range(0, length, block):
        p.run(np.ascontiguousarray(get(off, min(block, length - off))))
    return p


def _check_programme(out, i, p):
    want = p.ebu.read()[0]
    names = {"integrated": 4, "integ_thr": 5, "range_min": 6, "range_max": 7, "maxloudn_M": 1, "maxloudn_S": 3}
    for name, k in names.items():
        assert u32(out[name][i]) == u32(want[k]), (i, name, out[name][i], want[k])
    assert u32(out["tp_max"][i]) == u32(p.hold), (i, out["tp_max"][i], p.hold)


@pytest.mark.parametrize("nclips,nchan,layout", [(48, 2, None), (12, 6, "5.1")])
def test_programme_loudness_matches_private_instances(nclips, nchan, layout):
    import meters_lv2_b200 as B
    fs, block = 48000.0, 1024
    g = _gains(layout)
    rng = np.random.default_rng(nclips)
    ln = rng.integers(int(0.2 * fs), int(40 * fs), size=nclips)
    ln[0::5] = (ln[0::5] // block) * block                  # on a block edge
    ln[1::5] = (ln[1::5] // 2400) * 2400                    # on a fragment edge
    ln[2::5] = (ln[2::5] // 24000) * 24000 + 1              # one past an S-histogram period
    get = lambda off, n: np.concatenate([_clip(nclips, i, off, n, nchan, fs) for i in range(nclips)])
    out = B.programme_loudness(get, ln, fs, nchan=nchan, gains=g, block=block)
    for i in range(nclips):
        own = lambda off, n, i=i: _clip(nclips, i, off, n, nchan, fs)
        _check_programme(out, i, _private_programme(own, i, int(ln[i]), nchan, g, fs, block))


def test_programme_loudness_many_clips_on_device():
    """1024 stereo clips generated block by block on the device; a sampled subset against private instances"""
    import torch
    import meters_lv2_b200 as B
    fs, block, nclips, nchan = 48000.0, 1024, 1024, 2
    rng = np.random.default_rng(1024)
    ln = rng.integers(int(2 * fs), int(20 * fs), size=nclips)
    sample = rng.choice(nclips, size=10, replace=False)
    rows_s = np.concatenate([np.arange(i * nchan, (i + 1) * nchan) for i in sample])
    kept = {}
    freq = torch.arange(nclips * nchan, device="cuda", dtype=torch.float32)[:, None] * 3.0 + 60.0
    lvl = 10.0 ** (-2.0 * ((torch.arange(nclips * nchan, device="cuda") // nchan) % 11).float()[:, None] / 10.0)

    def gen(off, n):
        gcu = torch.Generator(device="cuda"); gcu.manual_seed(off)
        t = (off + torch.arange(n, device="cuda", dtype=torch.float64)) / fs
        x = (torch.randn(nclips * nchan, n, device="cuda", generator=gcu) * 0.2
             + 0.3 * torch.sin(2 * np.pi * freq.double() * t).float()) * lvl
        kept[off] = x[rows_s].cpu().numpy()
        return x

    out = B.programme_loudness(gen, ln, fs, nchan=nchan, block=block)
    for k, i in enumerate(sample):
        own = lambda off, n, k=k: kept[off][k * nchan:(k + 1) * nchan, :n]
        _check_programme(out, int(i), _private_programme(own, int(i), int(ln[i]), nchan, None, fs, block))


def test_zero_padding_changes_the_answer():
    """the same short clips zero-padded to the longest one (today's only option) report other maximum S loudness or range than the
    clips themselves; the ragged run is the private instance's answer"""
    import meters_lv2_b200 as B
    fs, block, nchan = 48000.0, 1024, 2
    ln = np.array([int(12.31 * fs), int(4.71 * fs), int(21.13 * fs), int(40 * fs)])      # ending inside a 50 ms fragment
    rows = len(ln) * nchan
    x = np.random.default_rng(3).standard_normal((rows, int(ln.max()))).astype(np.float32) * 0.5
    for i, n in enumerate(ln):
        x[i * nchan:(i + 1) * nchan, :n] *= (0.02 + (np.arange(n) / n) ** 2).astype(np.float32)   # a crescendo up to the clip's end
        x[i * nchan:(i + 1) * nchan, n:] = 0.0
    rag = B.programme_loudness(x, ln, fs, block=block)
    pad = B.programme_loudness(x, np.full(len(ln), ln.max()), fs, block=block)
    for i in range(len(ln)):
        own = lambda off, n, i=i: x[i * nchan:(i + 1) * nchan, off:off + n]
        _check_programme(rag, i, _private_programme(own, i, int(ln[i]), nchan, None, fs, block))
    diff = [(rag["maxloudn_S"][i] != pad["maxloudn_S"][i]) or (rag["range_min"][i] != pad["range_min"][i])
            or (rag["range_max"][i] != pad["range_max"][i]) for i in range(len(ln) - 1)]
    assert all(diff), (rag, pad)
