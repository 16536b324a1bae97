"""GPU parity at the edges: other sample rates, bank sizes that are not multiples of the kernels' tile sizes,
block lengths 1 and 8192 (the reference's maximum, jmeters/truepeakdsp.cc:44), one-instance banks."""
import numpy as np
import pytest

import _oracle as O
import _signals as S

pytestmark = pytest.mark.gpu
RES = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("fs,n_inst,blocks", [
    (44100.0, 1, [1024] * 150),            # fragment = 2205 frames: never aligned with the 1024 block
    (96000.0, 33, [1024] * 40 + [8192] * 8),
    (48000.0, 130, [1] * 5 + [8192] * 3 + [2400] * 4 + [2399, 2401]),
    (22050.0, 3, [512] * 200),
    (4000.0, 7, [8192] * 4 + [1] + [8192] * 4 + [3, 4097]),   # fragment = 200 frames: 41 fragment edges in 8192 frames, more than
                                                               # K1's 32 pieces per launch; after the 1-frame block the second
                                                               # launch starts at an unaligned offset
])
def test_ebu_rates_and_sizes(fs, n_inst, blocks):
    import torch
    import meters_lv2_b200 as B
    x = S.white(2 * n_inst, sum(blocks), seed=int(fs) % 1000)
    g = B.Ebu_r128_proc(n_inst, 2, fs); o = O.Ebu(n_inst, 2, fs)
    g.integr_start(); o.integr("start")
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for n in blocks:
        g.process(xd[:, pos:pos + n]); o.process(np.ascontiguousarray(x[:, pos:pos + n]), nthreads=8)
        pos += n
    gr, orr = g.results(), o.read()
    for i, name in enumerate(RES):
        assert np.array_equal(u32(gr[name]), u32(orr[:, i])), name
    for inst in {0, n_inst - 1}:
        hm, hs = g.histogram(inst); om, os_, oc = o.hist(inst)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_)
        z, pw, fr, c = g.state(inst); oz, opw, ofr, oc4 = o.state(inst)
        assert np.array_equal(u32(z), u32(oz)) and np.array_equal(u32(pw), u32(opw)) and list(c) == list(oc4)


@pytest.mark.parametrize("fs,C,blocks", [
    (44100.0, 1, [1024] * 12),
    (96000.0, 17, [8192] * 3 + [1] * 7 + [4] * 3),
    (48000.0, 129, [1024] * 6 + [1000, 24, 2, 6]),
    (192000.0, 7, [4096] * 4),
])
def test_truepeak_kmeter_rates_and_sizes(fs, C, blocks):
    import torch
    import meters_lv2_b200 as B
    x = S.white(C, sum(blocks), seed=int(fs) % 997)
    xd = torch.from_numpy(x).cuda()
    for mode in (0, 1):
        g = B.TruePeakKmeter(C, fs); ot = O.TruePeak(C, fs); ok = O.Kmeter(C, fs)
        pos = 0
        for bi, n in enumerate(blocks):
            blk = np.ascontiguousarray(x[:, pos:pos + n])
            g.process(xd[:, pos:pos + n], tp_mode=mode); ot.process(blk, mode=mode, nthreads=8); ok.process(blk, nthreads=8)
            pos += n
            if bi % 2 == 0:
                r = g.read(); m, p = ot.read(); rms, pk = ok.read()
                assert np.array_equal(u32(r["tp_m"]), u32(m)) and np.array_equal(u32(r["tp_p"]), u32(p)), (mode, bi)
                assert np.array_equal(u32(r["km_rms"]), u32(rms)) and np.array_equal(u32(r["km_peak"]), u32(pk)), (mode, bi)
        s = g.state(); m, p, z1, z2, res = ot.peek()
        assert np.array_equal(u32(s["z1"]), u32(z1)) and np.array_equal(u32(s["z2"]), u32(z2)) and np.array_equal(s["res"], res)
        assert np.array_equal(u32(s["km"]), u32(ok.peek()))


@pytest.mark.parametrize("fs,n_inst", [(44100, 1), (96000, 33), (48000, 65)])
def test_stcorr_rates_and_sizes(fs, n_inst):
    import torch
    import meters_lv2_b200 as B
    blocks = [1024] * 5 + [1, 8192, 31]
    x = S.white(2 * n_inst, sum(blocks), seed=fs % 991)
    g = B.Stcorrdsp(n_inst, fs); o = O.Stcorr(n_inst, fs)
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for n in blocks:
        g.process(xd[:, pos:pos + n]); o.process(np.ascontiguousarray(x[:, pos:pos + n]), nthreads=4)
        pos += n
    assert np.array_equal(u32(g.state()), u32(o.peek())) and np.array_equal(u32(g.read()), u32(o.read()))


@pytest.mark.parametrize("rate,n_inst,nchan", [(44100.0, 1, 2), (96000.0, 5, 1), (48000.0, 7, 2)])
def test_spectr_rates_and_sizes(rate, n_inst, nchan):
    import torch
    import meters_lv2_b200 as B
    blocks = [1024] * 3 + [1, 8192, 333]
    x = S.white(nchan * n_inst, sum(blocks), seed=int(rate) % 983)
    g = B.Spectr30(n_inst, nchan, rate); o = O.Spectr30(n_inst, nchan, rate)
    xd = torch.from_numpy(x).cuda()
    pos = 0
    for n in blocks:
        g.process(xd[:, pos:pos + n]); o.process(np.ascontiguousarray(x[:, pos:pos + n]), nthreads=8)
        pos += n
    assert np.array_equal(u32(g.read()), u32(o.read()))
    z, v, m = g.state(n_inst - 1); oz, ov, om = o.state(n_inst - 1)
    assert np.array_equal(z.view(np.uint64), oz.view(np.uint64)) and np.array_equal(u32(v), u32(ov)) and np.array_equal(u32(m), u32(om))


def test_block_length_limits_are_codes():
    import torch
    import meters_lv2_b200 as B
    x = torch.zeros((2, 9000), device="cuda")
    g = B.Ebu_r128_proc(1, 2)
    with pytest.raises(B.B200MError):
        g.process(x[:, :8193])                       # > 8192: the reference asserts (compiled out); here an error code
    with pytest.raises(B.B200MError):
        g.process_ptr(x.data_ptr(), 9000, 0)
    g.process(x[:, :8192])
