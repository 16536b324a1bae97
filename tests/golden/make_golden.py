"""Generates tests/golden/golden_v1.npz from the REFERENCE build (oracle/_ref, i.e. the unmodified
x42/meters.lv2 sources compiled by oracle/Makefile) on small seeded streams.

    python tests/golden/make_golden.py            # rewrite the fixture (needs /root/reference -> oracle/_ref)

The reference ships no golden vectors or tests (SURVEY.md §4), so these fixtures — outputs of the
reference itself, run here — are the pin for the oracle port on machines where /root/reference is absent.
`compute(kind)` is also what tests/test_oracle_port.py::test_golden_vectors replays.
The phasewheel entries come from the port (FFTW3 is absent: that path has no reference build).
It also writes ebur128_plugin.npz and goniometer_ref.npz (the reference side of two GPU tests) and ebu_hist_calc.npz (the
reference's calc_integ / calc_range on the synthetic histograms of tests/test_ebu_gating_gpu.py).  lv2_ref.npz, what the
reference's LV2 plugins write to their ports in the GPU tests, is recorded by those tests on a GPU machine with oracle/_ref built:
    B200M_LV2_REF_RECORD=$PWD/tests/golden/lv2_ref.npz python -m pytest -m gpu tests/test_lv2_*.py tests/test_dr14_gpu.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _oracle as O          # noqa: E402
import _signals as S         # noqa: E402

BLOCKS = [1024] * 130 + [480, 64, 8192, 1, 3, 1023]


def compute(kind):
    out = {}
    kind_o = kind
    x = S.white(8, sum(BLOCKS), seed=0xC0FFEE)
    x[6, 5000:5010] = [np.nan, np.inf, -np.inf, 1e-42, 0, 1, -1, 1e-30, 3e38, -3e38]
    e = O.Ebu(4, 2, kind=kind); e.integr("start")
    tp = O.TruePeak(8, kind=kind); km = O.Kmeter(8, kind=kind); co = O.Stcorr(4, kind=kind)
    sp = O.Spectr30(2, 2, kind=kind)
    tpm, kmr, cor = [], [], []
    pos = 0
    for i, n in enumerate(BLOCKS):
        blk = np.ascontiguousarray(x[:, pos:pos + n]); pos += n
        e.process(blk); tp.process(blk); km.process(blk); co.process(blk)
        if i < 24:
            sp.process(np.ascontiguousarray(blk[:4]))
        m, p = tp.read(); r, pk = km.read()
        tpm.append(np.stack([m, p])); kmr.append(np.stack([r, pk])); cor.append(co.read())
    out["ebu_results"] = e.read()
    for i in range(4):
        hm, hs, c = e.hist(i)
        out["ebu_histM_%d" % i], out["ebu_histS_%d" % i], out["ebu_counts_%d" % i] = hm, hs, c
    out["ebu_coeffs"] = e.coeffs()
    out["tp_reads"] = np.stack(tpm); out["km_reads"] = np.stack(kmr); out["cor_reads"] = np.stack(cor)
    w, t = tp.coeffs(); out["tp_w"], out["tp_ctab"] = w, t
    out["tp_upsampled"] = O.tp_upsample(x[0, :2048], kind=kind)
    ports = sp.read()
    out["spec_ports"] = ports[:, :30].copy(); out["spec_maxports"] = ports[:, 30:].copy()
    out["spec_coeffs"] = sp.coeffs()
    # needle-meter ballistics (VU, IEC I, IEC II, M/S PPM)
    for nk in range(4):
        nm = O.Needle(4, nk, oracle=kind_o)
        reads = []
        pos2 = 0
        for i, n in enumerate(BLOCKS[:40]):
            blk = np.ascontiguousarray((x[:8 if nk == 3 else 4, pos2:pos2 + n] * np.float32(3.0))); pos2 += n
            nm.process(blk); reads.append(nm.read())
        out["needle_reads_%d" % nk] = np.stack(reads)
        out["needle_state_%d" % nk] = nm.peek()
    # bit-meter (cumulative mode) and signal distribution histogram
    bm = O.Bitmeter(4, oracle=kind_o); bm.mode(1)
    sd = O.SigDist(4, oracle=kind_o); sd.integrate(True)
    pos3 = 0
    for n in BLOCKS[:30]:
        blk = np.ascontiguousarray(x[4:8, pos3:pos3 + n]); pos3 += n
        bm.process(blk); sd.process(blk)
    for i in (0, 2):
        h, c, mm, it = bm.read(i)
        out["bim_hist_%d" % i], out["bim_cnt_%d" % i], out["bim_minmax_%d" % i] = h, c, mm
        h, mp, av, it = sd.read(i)
        out["sdh_hist_%d" % i], out["sdh_maxpeak_%d" % i], out["sdh_stats_%d" % i] = h, mp, av
    # 997 Hz / -23 dBFS tone (EBU Tech 3341 case 1)
    s = S.sine(1024 * 300, 997.0, amp=10 ** (-23 / 20)); y = np.ascontiguousarray(np.stack([s, s]))
    e2 = O.Ebu(1, 2, kind=kind); e2.integr("start")
    for b in range(300):
        e2.process(np.ascontiguousarray(y[:, b * 1024:(b + 1) * 1024]))
    out["ebu_tone_results"] = e2.read()
    # DR-14 (stereo, 36 s in 8192-frame blocks: 12 scored windows) and TPnRMS (mono)
    t = np.arange(8192 * 212) / 48000.0
    env = (0.2 + 0.8 * np.abs(np.sin(2 * np.pi * t / 6.1))).astype(np.float32)
    xd = (S.white(4, 8192 * 212, seed=0xD214) * env * np.float32(2.5)).astype(np.float32)
    xd[2:4, 8192 * 60:8192 * 110] = 0.0                                    # instance 1: 3 s windows of silence are not scored
    dr = O.Dr14(2, 2, 48000.0, True, kind=kind)
    reads = []
    for b in range(212):
        dr.process(np.ascontiguousarray(xd[:, b * 8192:(b + 1) * 8192]))
        if b % 4 == 3:
            reads.append(dr.read())
        if b == 150:
            dr.reset()
    out["dr14_ports"] = np.stack(reads)
    tn = O.Dr14(3, 1, 44100.0, False, kind=kind)
    reads = []
    for b in range(40):
        tn.process(np.ascontiguousarray(x[:3, b * 1000:(b + 1) * 1000]))
        reads.append(tn.read())
    out["tpnrms_ports"] = np.stack(reads)
    # phasewheel (port only)
    pw = O.Phasewheel(2, 1024, kind="port")
    for b in range(4):
        pw.process(np.ascontiguousarray(x[:4, b * 1024:(b + 1) * 1024]))
    ph, lv, pk = pw.read()
    out["pw_phase"], out["pw_level"], out["pw_peak"] = ph, lv, pk
    return out


def ebur128_plugin_input():
    """the input of tests/test_ebu_gpu.py::test_r128_bank_vs_reference_ebur128_plugin: 10 stereo instances, 140 blocks"""
    x = S.white(2 * 10, 1024 * 140, seed=68)
    x[3] = 0
    return x


def ebur128_plugin_reads():
    """the reference's EBUr128 plugin (ebur128_run) on that input: its output ports after every 20th block, [7, 10, 10]"""
    x = ebur128_plugin_input()
    o = O.EbuPlugin(10, 48000.0, True)
    reads = []
    for b in range(140):
        o.run(np.ascontiguousarray(x[:, b * 1024:(b + 1) * 1024]), nthreads=8)
        if b % 20 == 19:
            reads.append(o.read())
    return np.stack(reads)


def ebu_hist_calc_reads(kind="reference"):
    """Ebu_r128_hist::calc_integ / calc_range of the reference on the synthetic histogram families of
    tests/test_ebu_gating_gpu.py: [n, 5] float32 (integrated, integ_thr, range_min, range_max, range_thr)"""
    import test_ebu_gating_gpu as GG
    return np.stack([O.hist_calc(hm, int(hm.sum()), hs, int(hs.sum()), kind=kind) for _, hm, hs in GG.hist_families()])


if __name__ == "__main__":
    assert O.available("reference"), "build oracle/_ref first (make -C oracle ref)"
    d = compute("reference")
    np.savez_compressed(os.path.join(HERE, "golden_v1.npz"), **d)
    print("wrote golden_v1.npz:", {k: v.shape for k, v in d.items()})
    np.savez_compressed(os.path.join(HERE, "ebur128_plugin.npz"), reads=ebur128_plugin_reads())
    print("wrote ebur128_plugin.npz")
    import test_lv2_gon_gpu as GON
    feed, rings = GON.reference_feed()
    state = GON.reference_saved_state()
    d = dict(layout=np.array([GON._layout(O.load("reference"), "refgon_layout")[k] for k in GON.FIELDS], np.int64),
             feed=feed, feed_rings=np.array(rings), state_keys=np.array(list(state), dtype=object).astype(bytes),
             state_types=np.array([v[1] for v in state.values()]), state_flags=np.array([v[2] for v in state.values()], np.int64))
    for i, v in enumerate(state.values()):
        d["state_value_%d" % i] = np.frombuffer(v[0], np.uint8)
    np.savez_compressed(os.path.join(HERE, "goniometer_ref.npz"), **d)
    print("wrote goniometer_ref.npz")
    np.savez_compressed(os.path.join(HERE, "ebu_hist_calc.npz"), out5=ebu_hist_calc_reads())
    print("wrote ebu_hist_calc.npz")
