"""GPU: per-instance 50 ms fragment clocks in the EBU R128 bank (csrc/ebu.cu, csrc/ebu_kw.cuh).

Instances of one bank are reset one by one (b200m_ebu_reset (h, inst), B200M_R128_NEW) at scripted blocks, so that many fragment
phases coexist inside one K1 warp.  After EVERY block each instance must equal, bit for bit, a reference Ebu_r128_proc reset at the
same points: the nine loudness floats, the last fragment power, both 751-bin histograms and their counts, and the instance's own
{frcnt, wrind, div1, div2}.
"""
import numpy as np
import pytest

import _oracle as O
from test_r128_fused_gpu import _Trio, _signal, u32

pytestmark = pytest.mark.gpu
RES = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")
SIZES = [1, 4, 1000, 2399, 2400, 2401, 8192]


def _program(rng, rows, n, nchan):
    """noise at a per-instance level that moves from block to block (the histograms spread over many bins)"""
    lvl = 10.0 ** rng.uniform(-3.0, 0.0, size=(rows // nchan, 1))
    return (rng.standard_normal((rows, n)) * np.repeat(lvl, nchan, axis=0)).astype(np.float32)


def _script(n_inst, nblk, seed):
    """{block: [(cmd, inst), ...]} with cmd in reset / start / pause / ireset; instance 0 is only ever started"""
    rng = np.random.default_rng(seed)
    script = {0: [("start", -1)]}
    for i in range(1, n_inst):
        for b in rng.choice(np.arange(1, nblk), 2, replace=False):
            script.setdefault(int(b), []).append(("reset", i))
            script[int(b)].append(("start", i))
        b = int(rng.integers(1, nblk))
        script.setdefault(b, []).append((str(rng.choice(["pause", "ireset", "start"])), i))
    return script


def _check_ebu(tag, eb, res, o, n_inst):
    """eb: the bank's Ebu_r128_proc view; res: its results; o: the reference bank"""
    orr = o.read()
    for k, name in enumerate(RES):
        bad = np.nonzero(u32(res[name]) != u32(orr[:, k]))[0]
        assert bad.size == 0, (tag, name, bad[:5], res[name][bad[:3]], orr[bad[:3], k])
    for i in range(n_inst):
        hm, hs = eb.histogram(i)
        om, os_, oc = o.hist(i)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_), (tag, i)
        assert res["hist_M_count"][i] == oc[0] and res["hist_S_count"][i] == oc[1], (tag, i)
        z, pw, fr, c = eb.state(i)
        oz, opw, ofr, oc4 = o.state(i)
        assert list(c) == list(oc4), (tag, i, list(c), list(oc4))
        assert np.array_equal(u32(z), u32(oz)) and np.array_equal(u32(pw), u32(opw)), (tag, i)
        assert u32(np.float32(fr)) == u32(np.float32(ofr)), (tag, i)
        assert u32(np.float32(res["frag_power"][i])) == u32(np.float32(opw[(oc4[1] - 1) & 63])) or oc4[1] == 0, (tag, i)


def _apply(script_b, g_reset, g_integr, o):
    for cmd, inst in script_b:
        if cmd == "reset":
            g_reset(inst); o.reset(inst)
        else:
            g_integr(cmd, inst)
            o.integr({"ireset": "reset"}.get(cmd, cmd), inst)


@pytest.mark.parametrize("fs", [48000.0, 44100.0, 4000.0])
@pytest.mark.parametrize("nchan,n_inst", [(1, 70), (2, 40), (5, 20)])
def test_phases_bit_exact_every_block(nchan, n_inst, fs):
    """device path, ragged blocks 1 .. 8192 frames; at 4 kHz an 8192-frame block completes ~41 fragments per instance and its
    S periods wrap at different fragments of the block for different instances"""
    import torch
    import meters_lv2_b200 as B
    rng = np.random.default_rng(int(fs) + nchan)
    sizes = list(rng.permutation(SIZES * 4))
    script = _script(n_inst, len(sizes), seed=nchan)
    g = B.Ebu_r128_proc(n_inst, nchan, fs)
    o = O.Ebu(n_inst, nchan, fs)
    fn = {"start": g.integr_start, "pause": g.integr_pause, "ireset": g.integr_reset}
    for b, n in enumerate(sizes):
        _apply(script.get(b, []), g.reset, lambda c, i: fn[c](i), o)
        x = _program(rng, n_inst * nchan, int(n), nchan)
        o.process(x, nthreads=8)
        g.process(torch.from_numpy(x).cuda())
        _check_ebu((b, n), g, g.results(), o, n_inst)
    assert len({int(g.state(i)[3][0]) for i in range(n_inst)}) > 4      # many phases at the end


def test_sliced_host_path_phases():
    """the EBUr128 bank's sliced host path: 70 instances in 4 slices whose bounds (17, 35, 52 instances) fall inside K1 warps;
    B200M_R128_NEW restarts an instance's clock"""
    import meters_lv2_b200 as B
    E = B.EBUr128
    n_inst = 70
    rng = np.random.default_rng(11)
    sizes = list(rng.permutation(SIZES * 3))
    script = _script(n_inst, len(sizes), seed=12)
    r = E(n_inst, 48000.0, dbtp_enable=True)
    o = O.Ebu(n_inst, 2, 48000.0)
    code = {"start": E.START, "pause": E.PAUSE, "ireset": E.RESET}     # RESET: integr_reset (+ the dBTP hold, not compared here)
    for b, n in enumerate(sizes):
        _apply(script.get(b, []), lambda i: r.control(E.NEW, i), lambda c, i: r.control(code[c], i), o)
        x = _program(rng, 2 * n_inst, int(n), 2)
        o.process(x, nthreads=8)
        r.run(x)
        res, _ = r.results()
        _check_ebu((b, n), r.ebu, res, o, n_inst)


def test_fused_path_many_phases():
    """6400 stereo instances in tolerance mode, 64 staggered phases (every 64th instance gets B200M_R128_NEW after each of 64
    warm-up blocks, so every K1 warp holds 16 phases): the fused kernel still replaces K1 + the FIR in every
    1024-frame cycle; EBU floats and histograms bit-identical to the exact bank and to the reference on a subset; dBTP within
    1e-4 dB of the exact bank"""
    import torch
    n_inst, n_ref = 6400, 128
    rng = np.random.default_rng(21)
    host = [_signal(rng, n_inst, 1024, i * 1024) for i in range(4)]
    dev = [torch.from_numpy(h).cuda() for h in host]
    tri = _Trio(n_inst, n_ref=0)
    o = O.Ebu(n_ref, 2, 48000.0)
    o.integr("start")
    for j in range(64):
        lf, le = tri.run(dev[j % 4], host[j % 4])
        assert le - lf == 1, (j, lf, le)
        o.process(np.ascontiguousarray(host[j % 4][:2 * n_ref]), nthreads=8)
        for i in range(j, n_ref, 64):
            o.reset(i); o.integr("start", i)
        for i in range(j, n_inst, 64):
            tri.control(tri.B.EBUr128.NEW, i)
        tri.control(tri.B.EBUr128.START, -1)
    for b in range(64, 330):
        lf, le = tri.run(dev[b % 4], host[b % 4])
        assert le - lf == 1, (b, lf, le)
        o.process(np.ascontiguousarray(host[b % 4][:2 * n_ref]), nthreads=8)
        if b % 49 == 0 or b == 329:
            rf, tf = tri.check(b)
            _, te = tri.exact.results()
            fin = np.isfinite(te)
            assert np.array_equal(np.isfinite(tf), fin)
            assert np.abs(tf[fin].astype(np.float64) - te[fin]).max() <= 1e-4
            orr = o.read()
            for k, name in enumerate(RES):
                assert np.array_equal(u32(rf[name][:n_ref]), u32(orr[:, k])), (b, name)
            for i in range(0, n_ref, 9):
                hm, hs = tri.fused.histogram(i)
                om, os_, _ = o.hist(i)
                assert np.array_equal(hm, om) and np.array_equal(hs, os_), (b, i)
    r, _ = tri.fused.results()
    assert (r["integrated"] > -200).mean() > 0.9


def test_one_phase_launch_count():
    """a bank with one phase issues exactly the launches its block schedule implies: one K1 per block (48 kHz, <= 8192 frames),
    one K2a per completed fragment, one K2b per S-period wrap of the integrating bank; a bank-wide reset keeps one phase"""
    import torch
    import meters_lv2_b200 as B
    n_inst, fragm = 40, 2400
    g = B.Ebu_r128_proc(n_inst, 2, 48000.0)
    g.integr_start()
    rng = np.random.default_rng(3)
    t, frag = 0, 0
    for b, n in enumerate([1000, 2400, 1, 8192, 2399, 4, 4800, 1024] * 6):
        if b == 20:
            g.reset(); g.integr_start(); t, frag = 0, 0
        x = torch.from_numpy(_program(rng, 2 * n_inst, n, 2)).cuda()
        l0 = B.launch_count(); g.process(x); torch.cuda.synchronize(); got = B.launch_count() - l0
        nf = (t % fragm + n) // fragm
        wraps = sum(1 for k in range(frag + 1, frag + nf + 1) if k % 10 == 0)
        assert got == 1 + nf + wraps, (b, n, got, nf, wraps)
        t += n; frag += nf


def test_multi_phase_snapshot_restore_and_old_magic():
    """a snapshot taken mid-run on a bank with several phases continues bit-identically after restore; a blob in the format
    before per-instance phases (magic BE01) is rejected"""
    import torch
    import meters_lv2_b200 as B
    E = B.EBUr128
    n_inst = 96
    rng = np.random.default_rng(8)
    blocks = [(n, _signal(rng, n_inst, n, 0)) for n in [1000, 2401, 8192, 1024, 2400, 4] * 4]
    a = E(n_inst, 48000.0, True); a.control(E.START)
    for b, (n, x) in enumerate(blocks[:10]):
        a.run(torch.from_numpy(x).cuda())
        for i in range(b, n_inst, 10):
            a.control(E.NEW, i); a.control(E.START, i)
    snap = a.snapshot()
    for n, x in blocks[10:]:
        a.run(torch.from_numpy(x).cuda())
    r1, t1 = a.results()
    h1 = [a.histogram(i) for i in range(0, n_inst, 7)]
    a.restore(snap)
    for n, x in blocks[10:]:
        a.run(torch.from_numpy(x).cuda())
    r2, t2 = a.results()
    assert r1.tobytes() == r2.tobytes() and u32(t1).tobytes() == u32(t2).tobytes()
    for k, i in enumerate(range(0, n_inst, 7)):
        hm, hs = a.histogram(i)
        assert np.array_equal(hm, h1[k][0]) and np.array_equal(hs, h1[k][1])
    old = snap.copy()
    old[16:20] = np.frombuffer(np.uint32(0x42453031).tobytes(), np.uint8)      # the EBU blob's magic, after two u64 sizes
    with pytest.raises(B.B200MError):
        a.restore(old)
