"""GPU: the EBUr128 cycle for weighted banks of 1..32 channels (b200m_r128_create_weighted, csrc/ebu.cu + r128.cu).

The EBU side is checked against the weighted restatement of Ebu_r128_proc (tests/_ebu_weighted.cc, bit-identical to the reference
with the reference's weights: test_r128_weighted_cpu.py), the dBTP hold against one reference TruePeakdsp per channel with the
fold of src/ebulv2.cc:360-367 (the largest read() before coef_to_db).  The weights' meaning is checked against an independent float64
BS.1770-4 computation.
"""
import ctypes as C

import numpy as np
import pytest

import _ebu_weighted as W
import _oracle as O

pytestmark = pytest.mark.gpu
FS = 48000.0
HAVE_REF = O.available("reference")
RES = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")
DEFAULT = {1: [2.0], 2: [1, 1], 3: [1, 1, 1], 4: [1, 1, 1, 1.41], 5: [1, 1, 1, 1.41, 1.41]}
_libm = C.CDLL("libm.so.6")
_libm.log10f.restype = C.c_float
_libm.log10f.argtypes = [C.c_float]
R128F_MIN_CH = 10240                              # csrc/tpk.cu: the smallest bank the fused kernel takes


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _db(v):
    """coef_to_db (src/ebulv2.cc:227-230): 20.0 * log10f (val), the double product rounded to float"""
    return np.float32(-np.inf) if v == 0 else np.float32(20.0 * float(_libm.log10f(float(v))))


def _layouts():
    import meters_lv2_b200 as B
    w71 = B.bs1770_weights([30, -30, 0, 90, -90, 135, -135], [0] * 7)                          # 7.1 without its LFE
    w714 = B.bs1770_weights([30, -30, 0, 90, -90, 135, -135, 45, -45, 135, -135], [0] * 7 + [35] * 4)
    # 22.2 without its two LFEs: middle layer (10), upper layer (9), bottom front (3)
    az22 = [60, -60, 0, 180, 90, -90, 135, -135, 30, -30, 45, -45, 0, 0, 180, 90, -90, 135, -135, 0, 45, -45]
    el22 = [0] * 10 + [35, 35, 35, 90, 35, 35, 35, 35, 35, -20, -20, -20]
    w22 = B.bs1770_weights(az22, el22)
    w32 = np.float32([1.0, 1.41, 0.5, 1.0, 0.0, 2.0, 1.41, 1.0] * 4)
    return {"quad": np.float32([1, 1, 1.41, 1.41]), "7.1": w71, "7.1.4": w714, "22.2": w22, "32": w32,
            "5.1+lfe": np.float32([1, 1, 1, 0, 1.41, 1.41])}


def _signal(rng, n_inst, nchan, n, t0):
    """per-instance level (-70..0 dBFS, some instances silent), noise + a tone per channel, one loud channel per instance"""
    lvl = 10.0 ** rng.uniform(-3.5, 0.0, size=(n_inst, 1))
    lvl[::11] = 0.0
    tt = (t0 + np.arange(n)) / FS
    x = rng.standard_normal((nchan * n_inst, n)).astype(np.float32) * 0.2
    x += 0.4 * np.sin(2 * np.pi * (150.0 + 11.0 * np.arange(nchan * n_inst)[:, None]) * tt).astype(np.float32)
    x = x * np.repeat(lvl, nchan, axis=0)
    loud = np.arange(n_inst) * nchan + rng.integers(0, nchan, n_inst)
    x[loud] *= 1.5
    return x.astype(np.float32)


class _Ref:
    """oracle of a weighted bank: the weighted Ebu_r128_proc restatement, a reference TruePeakdsp set per instance, the dBTP fold"""

    def __init__(self, n_inst, gains):
        self.n, self.nc, self.g = n_inst, len(gains), gains
        self.ebu = W.Ebu(n_inst, gains, FS)
        self.tp = [O.TruePeak(self.nc, FS) for _ in range(n_inst)]
        self.hold = np.full(n_inst, -np.inf, np.float32)
        self.on = np.ones(n_inst, bool)

    def fresh_tp(self, i):
        self.tp[i] = O.TruePeak(self.nc, FS)
        self.hold[i] = -np.inf

    def run(self, x, insts=None, with_ebu=True):
        if with_ebu:
            self.ebu.process(x)
        for i in (range(self.n) if insts is None else insts):
            if not self.on[i]:
                self.hold[i] = -np.inf
                continue
            self.tp[i].process(np.ascontiguousarray(x[i * self.nc:(i + 1) * self.nc]), mode=1)
            m, _ = self.tp[i].read()
            t = m[0]
            for c in range(1, self.nc):
                t = t if t > m[c] else m[c]
            tp = _db(t)
            if tp > self.hold[i]:
                self.hold[i] = tp


def _check_vs_ref(tag, bank, ref, ebu_ok):
    r, tp = bank.results()
    want = ref.ebu.read()
    for k, name in enumerate(RES):
        assert np.array_equal(u32(r[name][ebu_ok]), u32(want[ebu_ok, k])), (tag, name)
    assert np.array_equal(u32(tp), u32(ref.hold)), (tag, np.nonzero(u32(tp) != u32(ref.hold))[0][:5])
    for i in np.nonzero(ebu_ok)[0]:
        hm, hs = bank.histogram(int(i)); om, os_, _ = ref.ebu.hist(int(i))
        assert np.array_equal(hm, om) and np.array_equal(hs, os_), (tag, i)
        assert r["hist_M_count"][i] == om.sum() and r["hist_S_count"][i] == os_.sum(), (tag, i)


def _snapshot(bk):
    """the bank's snapshot written into a zeroed buffer (the blob's alignment padding is never written)"""
    import meters_lv2_b200 as B
    n = B.lib().b200m_r128_snapshot_size(bk.h)
    buf = np.zeros(n, np.uint8)
    B._ck(B.lib().b200m_r128_snapshot(bk.h, B._np_ptr(buf), n, None))
    return buf


def _cuda_kernels(fa, fb):
    """names of the CUDA kernels that one call of fa and one call of fb launch, from ONE torch.profiler capture: the two calls are
    separated by a torch kernel (a marker) and the capture's kernels are cut there in time order.  A capture that lacks the marker
    recorded no GPU activity at all (CUPTI occasionally delivers none for a short session): it says nothing about fa or fb and is
    taken again, with one more call of each, at most three times."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    marker = torch.ones(1, device="cuda")
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            fa()
            torch.cuda.synchronize()
            marker.mul_(3.0)
            torch.cuda.synchronize()
            fb()
            torch.cuda.synchronize()
        ev = sorted((e for e in p.events() if str(e.device_type).endswith("CUDA") and "Memcpy" not in e.name and "Memset" not in e.name),
                    key=lambda e: e.time_range.start)
        cut = [i for i, e in enumerate(ev) if "at::native" in e.name]
        if cut:
            break
    assert len(cut) == 1, ("no valid profiler capture", [e.name for e in ev])
    a, b = [e.name for e in ev[:cut[0]]], [e.name for e in ev[cut[0] + 1:]]
    assert a and b, "the profiler saw the marker but no kernel of a cycle"
    return sorted(a), sorted(b)


@pytest.mark.parametrize("nchan,n_inst,prec", [(1, 37, 0), (2, 601, 1), (3, 401, 1), (4, 41, 0), (5, 2100, 1)])
def test_default_weights_are_the_nch_bank(nchan, n_inst, prec):
    """the reference's weights through b200m_r128_create_weighted: the bank b200m_r128_create_nch makes -- results, holds,
    histograms, snapshot bytes and the kernels of a cycle (5 x 2100: the fused kernel; 601, 401: the tensor-core FIR)"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    a, b = E(n_inst, FS, True, nchan=nchan), E(n_inst, FS, True, nchan=nchan, gains=DEFAULT[nchan])
    rng = np.random.default_rng(n_inst + nchan)
    for bk in (a, b):
        bk.set_precision(prec)
        bk.control(E.START)
    for k in range(10):
        x = torch.from_numpy(_signal(rng, n_inst, nchan, 1024, k * 1024)).cuda()
        if k == 4:
            for bk in (a, b):
                bk.set_dbtp(False, 3); bk.control(E.NEW, 5)
        if k in (2, 7):
            ka, kb = _cuda_kernels(lambda: a.run(x), lambda: b.run(x))
            assert ka == kb, (k, ka, kb)
        else:
            counts = []
            for bk in (a, b):
                l0 = B.launch_count(); bk.run(x); torch.cuda.synchronize(); counts.append(B.launch_count() - l0)
            assert counts[0] == counts[1], (k, counts)
        ra, ta = a.results(); rb, tb = b.results()
        assert ra.tobytes() == rb.tobytes() and u32(ta).tobytes() == u32(tb).tobytes(), k
    for i in (0, n_inst // 2, n_inst - 1):
        assert all(np.array_equal(p, q) for p, q in zip(a.histogram(i), b.histogram(i)))
    assert _snapshot(a).tobytes() == _snapshot(b).tobytes()


@pytest.mark.parametrize("layout,n_inst", [("quad", 37), ("7.1", 23), ("7.1.4", 13), ("22.2", 9), ("32", 5), ("5.1+lfe", 29)])
def test_exact_device_and_host_vs_oracle(layout, n_inst):
    """exact mode, odd bank sizes (instances straddle K-weighting warps and 8-channel true-peak groups), 200 ragged blocks,
    per-instance START / PAUSE / RESET / CLEAR / NEW and dBTP toggles; every EBU float, histogram, count and tp_max bit-identical
    to the oracle after every block, on the device path and on the host path"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _layouts()[layout]
    nchan = len(g)
    rng = np.random.default_rng(nchan * 1000 + n_inst)
    dev, host = E(n_inst, FS, True, nchan=nchan, gains=g), E(n_inst, FS, True, nchan=nchan, gains=g)
    banks = (dev, host)
    ref = _Ref(n_inst, g)
    # CLEAR keeps the fragment clock running: no restatement counterpart for its EBU part until a NEW resets the instance on both sides
    ebu_ok = np.ones(n_inst, bool)
    checked = 0                                   # instance-blocks whose EBU part was compared
    for bk in banks:
        bk.control(E.START)
    ref.ebu.integr("start")
    sizes = [1, 3, 64, 1000, 1024, 4097, 8192]
    t0 = 0
    for b in range(200):
        if b >= 2 and b % 3 == 0:
            i = int(rng.integers(n_inst))
            cmd = ("start", "pause", "reset", "clear", "new", "dbtp")[int(rng.integers(6))]
            if cmd == "dbtp":
                v = not ref.on[i]
                for bk in banks:
                    bk.set_dbtp(v, i)
                ref.on[i] = v
            else:
                code = {"start": E.START, "pause": E.PAUSE, "reset": E.RESET, "clear": E.CLEAR, "new": E.NEW}[cmd]
                for bk in banks:
                    bk.control(code, i)
                if cmd in ("start", "pause", "reset"):
                    ref.ebu.integr(cmd, i)
                if cmd == "reset":
                    ref.hold[i] = -np.inf
                if cmd == "new":
                    ref.ebu.reset(i)
                if cmd in ("clear", "new"):
                    ref.fresh_tp(i)
                ebu_ok[i] = cmd != "clear" and (ebu_ok[i] or cmd == "new")
        n = sizes[int(rng.integers(len(sizes)))]
        x = _signal(rng, n_inst, nchan, n, t0); t0 += n
        dev.run(torch.from_numpy(x).cuda()); host.run(x)
        ref.run(x)
        _check_vs_ref((b, n, "device"), dev, ref, ebu_ok)
        _check_vs_ref((b, n, "host"), host, ref, ebu_ok)
        checked += int(ebu_ok.sum())
    assert checked >= 0.3 * 200 * n_inst and not ref.on.all(), checked


def _close(tag, a, b):
    fin = np.isfinite(b)
    assert np.array_equal(np.isfinite(a), fin), tag
    if fin.any():
        d = np.abs(a[fin].astype(np.float64) - b[fin].astype(np.float64)).max()
        assert d <= 1e-4, (tag, d)


@pytest.mark.parametrize("layout,n_inst", [("7.1.4", 931), ("7.1", 1400)])
def test_tolerance_mode(layout, n_inst):
    """tolerance mode on the device path: 11 x 931 = 10241 channels (at the fused size: weighted banks take the two-kernel cycle,
    K1 + the tensor-core FIR behind it) and 7 x 1400 = 9800 (just below it); EBU outputs bit-identical to an exact bank, tp_max
    within 1e-4 dB of the reference hold"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _layouts()[layout]
    nchan = len(g)
    assert (nchan * n_inst >= R128F_MIN_CH) == (layout == "7.1.4")
    rng = np.random.default_rng(nchan)
    tol, exact = E(n_inst, FS, True, nchan=nchan, gains=g), E(n_inst, FS, True, nchan=nchan, gains=g)
    tol.set_precision(B.PREC_FMA)
    for bk in (tol, exact):
        bk.control(E.START)
    probe = sorted({0, 1, 2, n_inst // 3, n_inst // 2 + 1, n_inst - 2, n_inst - 1})
    ref = _Ref(len(probe), g) if HAVE_REF else None
    rows = np.concatenate([np.arange(i * nchan, (i + 1) * nchan) for i in probe])
    for k, n in enumerate([1024] * 6 + [4096, 1000, 1024, 2048]):
        x = _signal(rng, n_inst, nchan, n, k * 4096)
        if k == 5:
            for bk in (tol, exact):
                bk.set_dbtp(False, probe[1])
            if ref:
                ref.on[1] = False
        xd = torch.from_numpy(x).cuda()
        tol.run(xd); exact.run(xd)
        rt, tt = tol.results(); re, te = exact.results()
        assert rt.tobytes() == re.tobytes(), k
        _close(k, tt, te)
        if ref:
            ref.run(np.ascontiguousarray(x[rows]), with_ebu=False)
            _close((k, "reference"), tt[probe], ref.hold)
    for i in probe:
        assert all(np.array_equal(p, q) for p, q in zip(tol.histogram(i), exact.histogram(i)))


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("layout,n_inst", [("7.1.4", 67), ("7.1", 131)])
def test_sliced_host_path(layout, n_inst, prec, monkeypatch):
    """the host path with 1..8 slices: slice bounds split 22- and 28-channel K-weighting warps and 8-channel true-peak groups;
    results bit-identical to the device path in the same precision"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _layouts()[layout]
    nchan = len(g)
    rng = np.random.default_rng(n_inst * nchan + prec)
    blocks = [_signal(rng, n_inst, nchan, n, 0) for n in (1024, 1000, 4097, 64, 1024)]
    dev = E(n_inst, FS, True, nchan=nchan, gains=g)
    dev.set_precision(prec); dev.control(E.START)
    want = []
    for x in blocks:
        dev.run(torch.from_numpy(x).cuda())
        r, tp = dev.results()
        want.append((r.tobytes(), u32(tp).tobytes(), dev.histogram(n_inst - 1)))
    for nsl in (1, 2, 3, 5, 8):
        monkeypatch.setenv("B200M_R128_SLICES", str(nsl))
        host = E(n_inst, FS, True, nchan=nchan, gains=g)
        host.set_precision(prec); host.control(E.START)
        for k, x in enumerate(blocks):
            host.run(x)
            r, tp = host.results()
            assert r.tobytes() == want[k][0] and u32(tp).tobytes() == want[k][1], (nsl, k)
            hm, hs = host.histogram(n_inst - 1)
            assert np.array_equal(hm, want[k][2][0]) and np.array_equal(hs, want[k][2][1]), (nsl, k)
        host.close()


def test_snapshot_restore_and_refusals():
    """a weighted 7.1.4 bank snapshotted mid-run (mixed dBTP, several fragment phases) continues bit-identically after a restore;
    blobs of another channel count, other gains, and default / weighted blobs across the two kinds are refused"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _layouts()["7.1.4"]
    n_inst = 41
    rng = np.random.default_rng(11)
    xs = [torch.from_numpy(_signal(rng, n_inst, 11, 1024, k * 1024)).cuda() for k in range(4)]
    bk = E(n_inst, FS, True, nchan=11, gains=g)
    bk.control(E.START)
    snap = None
    for k in range(30):
        if k == 5:
            bk.set_dbtp(False, 7); bk.control(E.NEW, 9)
        if k == 12:
            snap = bk.snapshot()
        bk.run(xs[k % 4])
    first, tp1 = bk.results()
    bk.restore(snap)
    for k in range(12, 30):
        bk.run(xs[k % 4])
    again, tp2 = bk.results()
    assert first.tobytes() == again.tobytes() and u32(tp1).tobytes() == u32(tp2).tobytes()
    g2 = g.copy(); g2[0] = np.float32(1.0000001)
    other_gains = E(n_inst, FS, True, nchan=11, gains=g2)
    other_count = E(n_inst, FS, True, nchan=7, gains=_layouts()["7.1"])
    for donor, taker in ((other_gains, bk), (bk, other_gains), (other_count, bk), (bk, other_count)):
        with pytest.raises(B.B200MError):
            taker.restore(donor.snapshot())
    dflt5 = E(n_inst, FS, True, nchan=5)
    w5 = E(n_inst, FS, True, nchan=5, gains=[1, 1, 1, 1.41, 1.0])
    for donor, taker in ((dflt5, w5), (w5, dflt5)):
        with pytest.raises(B.B200MError):
            taker.restore(donor.snapshot())
    w5.restore(w5.snapshot()); dflt5.restore(dflt5.snapshot())


# ---- the weights' meaning against an independent float64 BS.1770-4 computation (K-filter of BS.1770-4 Table 1 / 2 at 48 kHz)
_K1 = ([1.53512485958697, -2.69169618940638, 1.19839281085285], [1.0, -1.69065929318241, 0.73248077421585])
_K2 = ([1.0, -2.0, 1.0], [1.0, -1.99004745483398, 0.99007225036621])


def _bs1770(x, g, n):
    """float64 loudness of the last n frames of one instance's rows x with weights g: -0.691 + 10 log10 sum g_i mean(y_i^2)"""
    from scipy.signal import lfilter
    y = lfilter(*_K2, lfilter(*_K1, x.astype(np.float64), axis=-1), axis=-1)
    return -0.691 + 10.0 * np.log10(np.sum(np.asarray(g, np.float64) * (y[:, -n:] ** 2).mean(axis=1)))


def test_weights_meaning_side_vs_front():
    """the same noise in Lss instead of L of a 7.1.4 instance reads 10 log10 (1.41) = 1.49 LU louder; momentary and short-term
    loudness within 0.01 LU of float64 BS.1770-4"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _layouts()["7.1.4"]
    rng = np.random.default_rng(3)
    nblk, n = 120, 4800                           # 12 s, whole 50 ms fragments
    w = (rng.standard_normal(nblk * n) * 0.1).astype(np.float32)
    x = np.zeros((2 * 11, nblk * n), np.float32)
    x[0] = w; x[11 + 3] = w                       # instance 0: L;  instance 1: Lss
    bk = E(2, FS, True, nchan=11, gains=g)
    bk.control(E.START)
    xd = torch.from_numpy(x).cuda()
    for b in range(nblk):
        bk.run(xd[:, b * n:(b + 1) * n])
    r, _ = bk.results()
    for i in (0, 1):
        xi = x[11 * i:11 * (i + 1)]
        assert abs(r["loudness_M"][i] - _bs1770(xi, g, 19200)) <= 0.01, (i, r["loudness_M"][i])
        assert abs(r["loudness_S"][i] - _bs1770(xi, g, 144000)) <= 0.01, (i, r["loudness_S"][i])
    d = 10.0 * np.log10(1.41)
    assert abs((r["loudness_M"][1] - r["loudness_M"][0]) - d) <= 0.01
    assert abs((r["loudness_S"][1] - r["loudness_S"][0]) - d) <= 0.01


def test_zero_gain_row_is_only_in_the_hold():
    """a zero-gain LFE row changes the loudness by nothing (bitwise) and the dBTP hold by its own peak"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    g = _layouts()["5.1+lfe"]
    rng = np.random.default_rng(4)
    nblk, n = 60, 4800
    x = (rng.standard_normal((6, nblk * n)) * 0.05).astype(np.float32)
    lfe = x.copy(); lfe[3] = 0.9 * np.sin(2 * np.pi * 60.0 * np.arange(nblk * n) / FS).astype(np.float32)
    quiet = x.copy(); quiet[3] = 0.0
    a, b = E(1, FS, True, nchan=6, gains=g), E(1, FS, True, nchan=6, gains=g)
    for bk in (a, b):
        bk.control(E.START)
    la, lb = torch.from_numpy(lfe).cuda(), torch.from_numpy(quiet).cuda()
    for k in range(nblk):
        a.run(la[:, k * n:(k + 1) * n]); b.run(lb[:, k * n:(k + 1) * n])
    ra, ta = a.results(); rb, tb = b.results()
    for name in RES:
        assert u32(ra[name]).tobytes() == u32(rb[name]).tobytes(), name
    assert abs(ra["loudness_M"][0] - _bs1770(lfe, g, 19200)) <= 0.01
    # the hold is the largest true peak of all six rows: the LFE's 0.9 sine (about -0.9 dBTP) over the -13 dBFS noise
    assert ta[0] > tb[0] + 6.0 and abs(ta[0] - 20.0 * np.log10(0.9)) <= 0.05, (ta, tb)
    if HAVE_REF:
        ref = _Ref(1, g)
        for k in range(nblk):
            ref.run(np.ascontiguousarray(lfe[:, k * n:(k + 1) * n]), with_ebu=False)
        assert u32(ta).tobytes() == u32(ref.hold).tobytes()


def test_invalid_arguments():
    """nchan 0 or 33, a negative, NaN or infinite gain, all gains zero: B200M_E_INVAL and *out left NULL"""
    import meters_lv2_b200 as B
    L = B.lib()
    bad = [(0, [1.0]), (33, [1.0] * 33), (3, [1.0, -1.0, 1.0]), (3, [1.0, np.nan, 1.0]), (3, [np.inf, 1.0, 1.0]),
           (4, [0.0] * 4), (2, [-0.5, 0.0])]
    for nchan, gains in bad:
        gg = np.ascontiguousarray(gains if gains else [1.0], np.float32)
        for create in ("r128", "ebu"):
            h = B._v(12345)
            if create == "r128":
                rc = L.b200m_r128_create_weighted(C.byref(h), 0, 3, nchan, B._np_ptr(gg), FS, 1)
            else:
                rc = L.b200m_ebu_create_weighted(C.byref(h), 0, 3, nchan, B._np_ptr(gg), FS)
            assert rc == -1 and not h.value, (create, nchan, gains, rc)
    with pytest.raises(B.B200MError):
        B.EBUr128(4, FS, True, nchan=6)                # b200m_r128_create_nch still stops at 5
