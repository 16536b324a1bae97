"""GPU: per-instance dBTP in the EBUr128 bank (b200m_r128_set_dbtp_inst, csrc/r128.cu).

Instances switch dBTP on and off on scripts of their own.  A disabled instance runs no process_max (src/ebulv2.cc:344-347): its
two TruePeakdsp histories stay frozen, its hold is -inf after every disabled cycle (:365-366), and the first block after it is
re-enabled reads the samples that preceded the disable.  Reference: one pair of reference TruePeakdsp per instance that skips
process_max while disabled.  Exact mode must be bit-identical; tolerance mode (tensor-core FIR, fused kernel, sliced host path)
within 1e-4 dB of the exact bank.
"""
import ctypes as C

import numpy as np
import pytest

import _oracle as O
from test_r128_fused_gpu import _signal, u32

pytestmark = pytest.mark.gpu
_libm = C.CDLL("libm.so.6")
_libm.log10f.restype = C.c_float
_libm.log10f.argtypes = [C.c_float]


def _db(v):
    """coef_to_db (src/ebulv2.cc:227-230): 20.0 * log10f (val), the double product rounded to float"""
    return np.float32(-np.inf) if v == 0 else np.float32(20.0 * float(_libm.log10f(float(v))))


class _RefTP:
    """reference TruePeakdsp pairs for a subset of instances, each skipping process_max while its dBTP is off"""

    def __init__(self, insts, fs=48000.0):
        self.insts = list(insts)
        self.tp = [O.TruePeak(2, fs) for _ in self.insts]
        self.hold = np.full(len(self.insts), -np.inf, np.float32)

    def run(self, x, on):
        for k, i in enumerate(self.insts):
            if on[i]:
                self.tp[k].process(np.ascontiguousarray(x[2 * i:2 * i + 2]), mode=1)
                m, _ = self.tp[k].read()
                t = _db(m[0] if m[0] > m[1] else m[1])
                if t > self.hold[k]:
                    self.hold[k] = t
            else:
                self.hold[k] = -np.inf


def _toggles(rng, n_inst, nblk):
    """per block: a list of (inst, on) or ("all", on); mixed blocks, and uniform all-off / all-on stretches"""
    sc = {}
    for b in range(1, nblk):
        sc[b] = [(int(i), bool(rng.random() < 0.5)) for i in rng.choice(n_inst, max(1, n_inst // 12), replace=False)]
    sc[9] = [("all", False)]; sc[10] = []; sc[11] = [("all", True)]
    sc[14] = [(i, False) for i in range(n_inst)]            # all off, one instance at a time: a uniform mask again
    sc[16] = [(3, True)]
    return sc


def _apply(sc, banks, on):
    for inst, v in sc:
        for bk in banks:
            bk.set_dbtp(v, -1 if inst == "all" else inst)
        if inst == "all":
            on[:] = v
        else:
            on[inst] = v


def _close(tag, a, b):
    fin = np.isfinite(b)
    assert np.array_equal(np.isfinite(a), fin), (tag, np.nonzero(np.isfinite(a) != fin)[0][:5])
    if fin.any():
        assert np.abs(a[fin].astype(np.float64) - b[fin]).max() <= 1e-4, tag


@pytest.mark.parametrize("n_inst", [24, 600])
def test_mixed_masks_exact_tc_and_host_path(n_inst):
    """600 instances = 1200 aligned channels: the tolerance bank takes the tensor-core FIR (PDL co-run on the device path);
    the host bank runs the sliced host path; blocks of 1024 frames with ragged ones in between"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    rng = np.random.default_rng(n_inst)
    exact, tol, host = (E(n_inst, 48000.0, True) for _ in range(3))
    tol.set_precision(B.PREC_FMA); host.set_precision(B.PREC_FMA)
    banks = (exact, tol, host)
    sub = sorted(set(range(0, n_inst, max(1, n_inst // 24))) | {3})
    ref = _RefTP(sub)
    on = np.ones(n_inst, bool)
    sizes = [1024] * 8 + [1000, 4, 8192, 1024, 1024, 2401] + [1024] * 16
    sc = _toggles(rng, n_inst, len(sizes))
    for b, n in enumerate(sizes):
        _apply(sc.get(b, []), banks, on)
        x = _signal(rng, n_inst, n, b * 1024)
        exact.run(torch.from_numpy(x).cuda()); tol.run(torch.from_numpy(x).cuda()); host.run(x)
        ref.run(x, on)
        _, te = exact.results(); _, tt = tol.results(); _, th = host.results()
        assert np.all(np.isneginf(te[~on])), b
        assert np.array_equal(u32(te[sub]), u32(ref.hold)), (b, te[sub][:6], ref.hold[:6])
        _close((b, "device tolerance"), tt, te)
        _close((b, "host tolerance"), th, te)
    assert not on.all() and on.any()


def test_fused_path_mixed_masks():
    """6400 stereo instances, tolerance mode: the fused kernel runs in every cycle, mixed masks included; snapshot / restore in a
    mixed state continues bit-identically"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    n_inst = 6400
    rng = np.random.default_rng(3)
    host = [_signal(rng, n_inst, 1024, i * 1024) for i in range(4)]
    dev = [torch.from_numpy(h).cuda() for h in host]
    fused, exact = E(n_inst, 48000.0, True), E(n_inst, 48000.0, True)
    fused.set_precision(B.PREC_FMA)
    sub = list(range(0, n_inst, 401)) + [3]
    ref = _RefTP(sub)
    on = np.ones(n_inst, bool)
    sc = _toggles(rng, n_inst, 40)
    snap = None
    for b in range(40):
        _apply(sc.get(b, []), (fused, exact), on)
        l0 = B.launch_count(); fused.run(dev[b % 4]); torch.cuda.synchronize(); lf = B.launch_count() - l0
        l0 = B.launch_count(); exact.run(dev[b % 4]); torch.cuda.synchronize(); le = B.launch_count() - l0
        assert le - lf == (1 if on.any() else 0), (b, lf, le)              # K1 + tpmax_kernel -> one fused kernel
        ref.run(host[b % 4], on)
        rf, tf = fused.results(); re, te = exact.results()
        assert rf.tobytes() == re.tobytes(), b
        assert np.array_equal(u32(te[sub]), u32(ref.hold)), b
        _close(b, tf, te)
        if b == 25:
            snap = fused.snapshot()
    first, tp1 = fused.results()
    fused.restore(snap)
    for b in range(26, 40):
        _apply(sc.get(b, []), (fused,), on.copy())
        fused.run(dev[b % 4])
    again, tp2 = fused.results()
    assert first.tobytes() == again.tobytes() and u32(tp1).tobytes() == u32(tp2).tobytes()


def test_uniform_mask_adds_no_launch():
    """a bank whose instances all share one dBTP setting, however it was set, launches what a bank switched as a whole
    launches; a mixed mask adds the fix-up kernel (and, in its first cycle, the stash kernel)"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    n_inst = 64
    x = torch.from_numpy(_signal(np.random.default_rng(1), n_inst, 1024, 0)).cuda()
    a, b = E(n_inst, 48000.0, True), E(n_inst, 48000.0, True)

    def launches(bank):
        l0 = B.launch_count(); bank.run(x); torch.cuda.synchronize()
        return B.launch_count() - l0
    for i in range(n_inst):
        a.set_dbtp(True, i)
    for _ in range(3):
        assert launches(a) == launches(b)
    for i in range(n_inst):
        a.set_dbtp(False, i)
    b.set_dbtp(False)
    for _ in range(3):
        assert launches(a) == launches(b)
    a.set_dbtp(True, 5); b.set_dbtp(True)
    assert launches(a) == launches(b) + 2
    for _ in range(3):
        assert launches(a) == launches(b) + 1
