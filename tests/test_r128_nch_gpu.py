"""GPU: the EBUr128 cycle for instances of 1..5 channels (b200m_r128_create_nch, csrc/r128.cu + csrc/tpk.cu).

The reference cycle is src/ebulv2.cc:341-367 with nchan channels: Ebu_r128_proc::process over the instance's rows, process_max on
each of its TruePeakdsp, t = the largest read() (taken before coef_to_db), tp_max = max (tp_max, coef_to_db (t)).  The oracle side
is composed of the reference's Ebu_r128_proc bank and one TruePeakdsp set per instance; coef_to_db runs through the host libm's
log10f like the reference.
 * 1 and 4 channels fold the hold inside each 8-channel true-peak group, 3 and 5 channels in r128_hold_kernel behind the groups;
 * the fused kernel cuts the bank into 128-channel (3, 5: 120-channel) slabs of whole instances.
"""
import ctypes as C

import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
FS = 48000.0
HAVE_REF = O.available("reference")
RES = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")
_libm = C.CDLL("libm.so.6")
_libm.log10f.restype = C.c_float
_libm.log10f.argtypes = [C.c_float]


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _db(v):
    """coef_to_db (src/ebulv2.cc:227-230): 20.0 * log10f (val), the double product rounded to float"""
    return np.float32(-np.inf) if v == 0 else np.float32(20.0 * float(_libm.log10f(float(v))))


def _signal(rng, n_inst, nchan, n, t0):
    """per-instance level (-70..0 dBFS, some instances silent), noise + a tone per channel, one loud channel per instance"""
    lvl = 10.0 ** rng.uniform(-3.5, 0.0, size=(n_inst, 1))
    lvl[::11] = 0.0
    tt = (t0 + np.arange(n)) / FS
    x = rng.standard_normal((nchan * n_inst, n)).astype(np.float32) * 0.2
    x += 0.4 * np.sin(2 * np.pi * (150.0 + 11.0 * np.arange(nchan * n_inst)[:, None]) * tt).astype(np.float32)
    x = x * np.repeat(lvl, nchan, axis=0)
    loud = np.arange(n_inst) * nchan + rng.integers(0, nchan, n_inst)       # the largest read moves between the channels
    x[loud] *= 1.5
    return x.astype(np.float32)


class _Ref:
    """oracle of a whole bank: the reference's Ebu_r128_proc bank, a TruePeakdsp set per instance and the dBTP fold"""

    def __init__(self, n_inst, nchan):
        self.n, self.nc = n_inst, nchan
        self.ebu = O.Ebu(n_inst, nchan, FS)
        self.tp = [O.TruePeak(nchan, FS) for _ in range(n_inst)]
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


@pytest.mark.skipif(not HAVE_REF, reason="needs the reference oracle (oracle/_ref)")
@pytest.mark.parametrize("nchan,n_inst", [(1, 37), (3, 37), (4, 41), (5, 41)])
def test_exact_device_and_host_vs_reference(nchan, n_inst):
    """exact mode, odd bank sizes (instances straddle 30/32-lane K-weighting warps and 8-channel true-peak groups), 200 ragged
    blocks, per-instance START / PAUSE / RESET / CLEAR / NEW and dBTP toggles; nine EBU floats, histograms, counts and tp_max
    bit-identical to the reference after every block, on the device path and on the sliced host path"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    rng = np.random.default_rng(100 + nchan)
    dev, host = E(n_inst, FS, True, nchan=nchan), E(n_inst, FS, True, nchan=nchan)
    banks = (dev, host)
    ref = _Ref(n_inst, nchan)
    ebu_ok = np.ones(n_inst, bool)                # CLEAR keeps the fragment clock running: no reference counterpart for its EBU part
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
                if cmd == "clear":
                    ebu_ok[i] = False
        n = sizes[int(rng.integers(len(sizes)))]
        x = _signal(rng, n_inst, nchan, n, t0); t0 += n
        dev.run(torch.from_numpy(x).cuda()); host.run(x)
        ref.run(x)
        _check_vs_ref((b, n, "device"), dev, ref, ebu_ok)
        _check_vs_ref((b, n, "host"), host, ref, ebu_ok)
    assert ebu_ok.sum() >= n_inst // 2 and not ref.on.all()


def _plain_stereo(n_inst):
    """a stereo bank made by b200m_r128_create itself"""
    import meters_lv2_b200 as B
    bk = B.EBUr128.__new__(B.EBUr128)
    B._Bank.__init__(bk)
    bk.n_inst, bk.nchan, bk.ebu = n_inst, 2, None
    B._ck(B.lib().b200m_r128_create(C.byref(bk.h), 0, n_inst, FS, 1))
    return bk


def _snapshot(bk):
    """the bank's snapshot written into a zeroed buffer (the blob's alignment padding is never written)"""
    import meters_lv2_b200 as B
    n = B.lib().b200m_r128_snapshot_size(bk.h)
    buf = np.zeros(n, np.uint8)
    B._ck(B.lib().b200m_r128_snapshot(bk.h, B._np_ptr(buf), n, None))
    return buf


@pytest.mark.parametrize("n_inst,prec", [(37, 0), (601, 1), (5120, 1)])
def test_stereo_nch_bank_is_the_stereo_bank(n_inst, prec):
    """nchan = 2 through b200m_r128_create_nch: the same results, snapshot bytes and launches per cycle as b200m_r128_create
    (37: tpmax_kernel; 601: tensor-core FIR; 5120: the fused kernel)"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    a, b = _plain_stereo(n_inst), E(n_inst, FS, True, nchan=2)
    rng = np.random.default_rng(n_inst)
    for bk in (a, b):
        bk.set_precision(prec)
        bk.control(E.START)
    for k in range(10):
        x = torch.from_numpy(_signal(rng, n_inst, 2, 1024, k * 1024)).cuda()
        if k == 4:
            for bk in (a, b):
                bk.set_dbtp(False, 3); bk.control(E.NEW, 5)
        counts = []
        for bk in (a, b):
            l0 = B.launch_count(); bk.run(x); torch.cuda.synchronize(); counts.append(B.launch_count() - l0)
        assert counts[0] == counts[1], (k, counts)
        ra, ta = a.results(); rb, tb = b.results()
        assert ra.tobytes() == rb.tobytes() and u32(ta).tobytes() == u32(tb).tobytes(), k
    assert _snapshot(a).tobytes() == _snapshot(b).tobytes()


def _edges(n_inst, nchan):
    """the first and last instance of every fused slab, and the bank's last instance"""
    per = 4 * (32 // nchan)                       # instances per slab
    s = set()
    for a in range(0, n_inst, per):
        s |= {a, min(a + per, n_inst) - 1}
    return sorted(s | {n_inst - 1})


def _close(tag, a, b):
    fin = np.isfinite(b)
    assert np.array_equal(np.isfinite(a), fin), tag
    if fin.any():
        d = np.abs(a[fin].astype(np.float64) - b[fin].astype(np.float64)).max()
        assert d <= 1e-4, (tag, d)


@pytest.mark.parametrize("nchan,n_inst", [(1, 10240), (3, 3414), (4, 2560), (5, 2100)])
def test_fused_tolerance_large_banks(nchan, n_inst):
    """tolerance mode, fused sizes: one fused kernel per cycle (as many launches as the stereo fused cycle), EBU floats and
    histograms bit-identical to an exact bank, tp_max bit-identical to the sliced host path (tensor-core FIR per slice) and within
    1e-4 dB of the reference on the instances at slab edges"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    rng = np.random.default_rng(nchan)
    fused, exact, host = (E(n_inst, FS, True, nchan=nchan) for _ in range(3))
    fused.set_precision(B.PREC_FMA); host.set_precision(B.PREC_FMA)
    for bk in (fused, exact, host):
        bk.control(E.START)
    edges = _edges(n_inst, nchan)
    ref = _Ref(n_inst, nchan) if HAVE_REF else None
    stereo = E(5120, FS, True)                     # the stereo fused cycle, in step (fragment ends add launches)
    stereo.set_precision(B.PREC_FMA); stereo.control(E.START)
    zeros = torch.zeros(10240, 1024, device="cuda")
    for k in range(12):
        x = _signal(rng, n_inst, nchan, 1024, k * 1024)
        xd = torch.from_numpy(x).cuda()
        if k == 6:
            for bk in (fused, exact, host):
                bk.set_dbtp(False, edges[1])
            if ref:
                ref.on[edges[1]] = False
        l0 = B.launch_count(); fused.run(xd); torch.cuda.synchronize(); lf = B.launch_count() - l0
        l0 = B.launch_count(); stereo.run(zeros); torch.cuda.synchronize(); ls = B.launch_count() - l0
        exact.run(xd); host.run(x)
        # a mixed dBTP mask adds the fix-up kernel, and its first cycle the stash kernel, to either cycle
        assert lf == ls + (0 if k < 6 else 2 if k == 6 else 1), (k, lf, ls)
        rf, tf = fused.results(); re, te = exact.results(); _, th = host.results()
        assert rf.tobytes() == re.tobytes(), k
        assert np.array_equal(u32(tf), u32(th)), (k, np.nonzero(u32(tf) != u32(th))[0][:5])
        _close(k, tf, te)
        if ref:
            ref.run(x, insts=edges, with_ebu=False)           # the EBU part is compared with the exact bank above
            _close((k, "reference"), tf[edges], ref.hold[edges])
    for i in edges[:8] + [n_inst - 1]:
        hf, sf = fused.histogram(i); he, se = exact.histogram(i)
        assert np.array_equal(hf, he) and np.array_equal(sf, se), i


@pytest.mark.parametrize("nchan,n_inst", [(1, 1200), (3, 401), (4, 301), (5, 241)])
def test_tensor_core_tolerance(nchan, n_inst):
    """tolerance mode below the fused size: the tensor-core FIR with the PDL co-run on the device path; EBU bit-identical, tp_max
    within 1e-4 dB of an exact bank"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    rng = np.random.default_rng(7 + nchan)
    tol, exact = E(n_inst, FS, True, nchan=nchan), E(n_inst, FS, True, nchan=nchan)
    tol.set_precision(B.PREC_FMA)
    for k, n in enumerate([1024] * 6 + [4096, 1000, 1024]):
        xd = torch.from_numpy(_signal(rng, n_inst, nchan, n, k * 4096)).cuda()
        tol.run(xd); exact.run(xd)
        rt, tt = tol.results(); re, te = exact.results()
        assert rt.tobytes() == re.tobytes(), k
        _close(k, tt, te)


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("nchan", [1, 2, 3, 4, 5])
def test_sliced_host_path(nchan, prec, monkeypatch):
    """the host path with 1..8 slices at 67 and 131 instances: slice bounds split K-weighting warps and true-peak groups; results
    bit-identical to the device path in the same precision"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    for n_inst in (67, 131):
        rng = np.random.default_rng(n_inst * nchan + prec)
        blocks = [_signal(rng, n_inst, nchan, n, 0) for n in (1024, 1000, 4097, 64, 1024)]
        dev = E(n_inst, FS, True, nchan=nchan)
        dev.set_precision(prec); dev.control(E.START)
        want = []
        for x in blocks:
            dev.run(torch.from_numpy(x).cuda())
            r, tp = dev.results()
            want.append((r.tobytes(), u32(tp).tobytes(), dev.histogram(n_inst - 1)))
        for nsl in (1, 2, 3, 5, 8):
            monkeypatch.setenv("B200M_R128_SLICES", str(nsl))
            host = E(n_inst, FS, True, nchan=nchan)
            host.set_precision(prec); host.control(E.START)
            for k, x in enumerate(blocks):
                host.run(x)
                r, tp = host.results()
                assert r.tobytes() == want[k][0] and u32(tp).tobytes() == want[k][1], (n_inst, nsl, k)
                hm, hs = host.histogram(n_inst - 1)
                assert np.array_equal(hm, want[k][2][0]) and np.array_equal(hs, want[k][2][1]), (n_inst, nsl, k)
            host.close()


def test_snapshot_restore_five_channels():
    """a 5-channel bank snapshotted mid-run (mixed dBTP) continues bit-identically after a restore; a stereo bank's blob is refused"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    n_inst = 41
    rng = np.random.default_rng(5)
    xs = [torch.from_numpy(_signal(rng, n_inst, 5, 1024, k * 1024)).cuda() for k in range(4)]
    bk = E(n_inst, FS, True, nchan=5)
    bk.control(E.START)
    snap = None
    for k in range(30):
        if k == 5:
            bk.set_dbtp(False, 7)
        if k == 12:
            snap = bk.snapshot()
        bk.run(xs[k % 4])
    first, tp1 = bk.results()
    bk.restore(snap)
    for k in range(12, 30):
        bk.run(xs[k % 4])
    again, tp2 = bk.results()
    assert first.tobytes() == again.tobytes() and u32(tp1).tobytes() == u32(tp2).tobytes()
    stereo = E(n_inst, FS, True)
    with pytest.raises(B.B200MError):
        bk.restore(stereo.snapshot())
    with pytest.raises(B.B200MError):
        E(4, FS, True, nchan=6)
