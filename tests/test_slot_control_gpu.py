"""GPU, through the C ABI: per-instance control of the spectrum bank, per-unit M/S gains of the needle-meter bank, and the per-slot
clears of the correlation, needle-meter and spectrum banks.  A bank instance driven with its own controls, or cleared in the middle
of a run, must read bit for bit what a bank of one driven the same way reads; every other instance must not notice."""
import numpy as np
import pytest

import _oracle as O
import _signals as S

pytestmark = pytest.mark.gpu

RAGGED = [1024, 1, 777, 64, 333, 2048, 5, 1000, 63, 512, 1536, 7]
SPEEDS = [1.0, 0.5, 3.0, 7.5, 15.0, 0.01, 0.004, 22.0, 2.0]          # 0.004 and 22 clamp at 0.01 / 15
RESETS = [0.0, 1.0, -1.0, 3.0, -3.0, -4.0, 3.0, 3.0, -3.0, -3.0]       # repeated +-3: the GUI's pending handshake


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def spec_script(n_inst, nblocks, seed):
    """[block][inst] (speed, reset): every instance changes its own controls at its own blocks"""
    rng = np.random.default_rng(seed)
    ctl = np.empty((nblocks, n_inst, 2), np.float32)
    cur = np.tile(np.float32([1.0, -4.0]), (n_inst, 1))
    for b in range(nblocks):
        for i in range(n_inst):
            if rng.random() < 0.3:
                cur[i, 0] = SPEEDS[rng.integers(len(SPEEDS))]
            if rng.random() < 0.35:
                cur[i, 1] = RESETS[rng.integers(len(RESETS))]
        ctl[b] = cur
    return ctl


def spec_ports_equal(got, want):
    """band levels bit for bit; maxima bit for bit except where the reference forces a GUI redraw (-500 - rand())"""
    assert np.array_equal(u32(got[..., :30]), u32(want[..., :30]))
    pend = want[..., 30:] <= -500
    assert np.array_equal(pend, got[..., 30:] <= -500)
    assert np.array_equal(u32(got[..., 30:][~pend]), u32(want[..., 30:][~pend]))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("n_inst,nchan", [(37, 1), (35, 2)])
@pytest.mark.parametrize("fma", [False, True])
def test_spec_per_instance_controls_equal_private_banks(n_inst, nchan, fma):
    """every instance with its own speed / reset script equals a bank of one driven through the bank-wide call; a subset also equals
    the reference's spectr30 (exact mode)"""
    import torch
    import meters_lv2_b200 as B
    x = S.white(n_inst * nchan, sum(RAGGED), seed=31 + nchan)
    xd = torch.from_numpy(x).cuda()
    ctl = spec_script(n_inst, len(RAGGED), seed=5 + nchan)
    g = B.Spectr30(n_inst, nchan)
    priv = [B.Spectr30(1, nchan) for _ in range(n_inst)]
    for bank in [g] + priv:
        bank.set_precision(B.PREC_FMA if fma else B.PREC_EXACT)
    oracle = [O.Spectr30(1, nchan) for _ in range(4)] if not fma else []
    pos = 0
    for b, n in enumerate(RAGGED):
        blk = np.ascontiguousarray(x[:, pos:pos + n])
        if nchan == 2:
            g.process(xd[:, pos:pos + n], speed=ctl[b, :, 0], reset=ctl[b, :, 1])      # device path
        else:
            g.process(blk, speed=ctl[b, :, 0], reset=ctl[b, :, 1])                     # host path
        for i, p in enumerate(priv):
            p.process(np.ascontiguousarray(blk[i * nchan:(i + 1) * nchan]), speed=float(ctl[b, i, 0]), reset=float(ctl[b, i, 1]))
        for i, o in enumerate(oracle):
            o.process(np.ascontiguousarray(blk[i * nchan:(i + 1) * nchan]), float(ctl[b, i, 0]), float(ctl[b, i, 1]))
        pos += n
        got = g.read()
        for i, p in enumerate(priv):
            assert np.array_equal(u32(got[i]), u32(p.read()[0])), (b, i)
            z, v, m = g.state(i); pz, pv, pm = p.state(0)
            assert np.array_equal(u64(z), u64(pz)) and np.array_equal(u32(v), u32(pv)) and np.array_equal(u32(m), u32(pm)), (b, i)
        for i, o in enumerate(oracle):
            spec_ports_equal(got[i], o.read()[0])
    assert (ctl[:, :, 1] == 3).any() and (ctl[:, :, 0] == 22.0).any()


def test_spec_bank_wide_call_is_the_uniform_per_instance_call():
    """uniform arrays through the per-instance call equal the bank-wide call bit for bit; a bank-wide call launches one kernel and,
    while the controls stay constant, copies nothing to the device"""
    import torch
    import meters_lv2_b200 as B
    from torch.profiler import ProfilerActivity, profile
    n_inst, nb = 70, 10
    x = torch.from_numpy(S.white(2 * n_inst, 1024 * nb, seed=8)).cuda()
    a, c = B.Spectr30(n_inst, 2), B.Spectr30(n_inst, 2)
    script = {0: (1.0, -4.0), 2: (3.0, -4.0), 4: (3.0, 1.0), 5: (3.0, 3.0), 6: (3.0, 3.0), 7: (0.5, -3.0)}
    spd, rst = 1.0, -4.0
    for b in range(nb):
        spd, rst = script.get(b, (spd, rst))
        blk = x[:, b * 1024:(b + 1) * 1024]
        l0 = B.launch_count()
        a.process(blk, speed=spd, reset=rst)
        assert B.launch_count() - l0 == 1
        c.process(blk, speed=np.full(n_inst, spd, np.float32), reset=np.full(n_inst, rst, np.float32))
        assert np.array_equal(u32(a.read()), u32(c.read())), b
        assert np.array_equal(u64(a.state(n_inst - 1)[0]), u64(c.state(n_inst - 1)[0])), b

    def h2d_copies(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return sum(1 for e in prof.events() if "memcpy" in e.name.lower() and "htod" in e.name.lower())

    blk = x[:, :1024]
    for _ in range(3):
        a.process(blk, speed=2.0, reset=-4.0)                 # the handshake fires and settles
    assert h2d_copies(lambda: [a.process(blk, speed=2.0, reset=-4.0) for _ in range(5)]) == 0
    assert h2d_copies(lambda: a.process(blk, speed=4.0, reset=-4.0)) == 1      # a change is uploaded once, as one copy


def _clear_run(make, feed, read, nunits, slots, blocks, clear_at, x_for):
    """bank `g` cleared at `slots` before block clear_at against an uncleared bank `u` and, per cleared slot, a fresh bank of one fed
    the slot's input from that block on"""
    g, u = make(nunits), make(nunits)
    fresh = {}
    pos = 0
    for b, n in enumerate(blocks):
        if b == clear_at:
            for s in slots:
                g.clear(s)
                fresh[s] = make(1)
        feed(g, x_for(slice(None), pos, n)); feed(u, x_for(slice(None), pos, n))
        for s, f in fresh.items():
            feed(f, x_for(s, pos, n))
        pos += n
        rg, ru = read(g), read(u)
        keep = np.setdiff1d(np.arange(nunits), list(fresh))
        for k in rg:
            assert np.array_equal(rg[k][keep].view(np.uint8), ru[k][keep].view(np.uint8)), (b, k)
            for s, f in fresh.items():
                assert np.array_equal(rg[k][[s]].view(np.uint8), read(f)[k][[0]].view(np.uint8)), (b, k, s)
        if b < clear_at:
            for k in rg:
                assert np.array_equal(rg[k].view(np.uint8), ru[k].view(np.uint8))
    return g


@pytest.mark.parametrize("fma", [False, True])
def test_cor_clear(fma):
    import torch
    import meters_lv2_b200 as B
    n = 70                                                   # exact: 3 warps of 32 pairs; FMA: 18 CTAs of 4 pairs
    blocks = RAGGED[:8]
    x = S.white(2 * n, sum(blocks), seed=41); x[1] = 0.7 * x[0] + 0.3 * x[1]
    xd = torch.from_numpy(x).cuda()

    def make(k):
        c = B.Stcorrdsp(k); c.set_precision(B.PREC_FMA if fma else B.PREC_EXACT)
        return c

    def x_for(s, pos, m):
        return xd[:, pos:pos + m] if isinstance(s, slice) else xd[2 * s:2 * s + 2, pos:pos + m]

    _clear_run(make, lambda c, blk: c.process(blk), lambda c: {"r": c.read(), "s": c.state()}, n, [0, 37, 69], blocks, 3, x_for)


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_ppm_clear(kind):
    import torch
    import meters_lv2_b200 as B
    n = 70                                                   # 3 warps of 32 units
    rows = 2 * n if kind == B.PPM_MS else n
    blocks = RAGGED[:8]
    x = S.white(rows, sum(blocks), seed=43) * np.float32(2.0)
    xd = torch.from_numpy(x).cuda()
    per = rows // n

    def make(k):
        m = B.NeedleMeters(k, kind)
        if kind == B.PPM_MS and k == n:
            m.set_gain(-6, 14, unit=37)                      # a cleared pair returns to the constructor's -6 / -6
        return m

    def x_for(s, pos, m):
        return xd[:, pos:pos + m] if isinstance(s, slice) else xd[per * s:per * s + per, pos:pos + m]

    def read(m):
        r, st = m.read(), m.state()
        return {"r": r.reshape(-1, per), "s": st.reshape(-1, per, 4)}

    _clear_run(make, lambda m, blk: m.process(blk), read, n, [0, 37, 69], blocks, 3, x_for)


@pytest.mark.parametrize("fma", [False, True])
def test_spec_clear(fma):
    import torch
    import meters_lv2_b200 as B
    n = 37                                                   # 10 CTAs of 4 instances, the last one partial
    blocks = RAGGED[:8]
    x = S.white(2 * n, sum(blocks), seed=47)
    xd = torch.from_numpy(x).cuda()
    ctl = spec_script(n, len(blocks), seed=9)

    def make(k):
        s = B.Spectr30(k, 2); s.set_precision(B.PREC_FMA if fma else B.PREC_EXACT)
        return s

    def read(s):
        z = np.stack([s.state(i)[0] for i in range(s.n_inst)]); vm = np.stack([np.concatenate(s.state(i)[1:]) for i in range(s.n_inst)])
        return {"p": s.read(), "z": z, "vm": vm}

    g, u = make(n), make(n)
    fresh = {}
    pos = 0
    for b, m in enumerate(blocks):
        if b == 3:
            for sl in (0, 17, 36):
                g.clear(sl)
                fresh[sl] = make(1)
        for bank in (g, u):
            bank.process(xd[:, pos:pos + m], speed=ctl[b, :, 0], reset=ctl[b, :, 1])
        for sl, f in fresh.items():
            f.process(xd[2 * sl:2 * sl + 2, pos:pos + m], speed=float(ctl[b, sl, 0]), reset=float(ctl[b, sl, 1]))
        pos += m
        rg, ru = read(g), read(u)
        keep = np.setdiff1d(np.arange(n), list(fresh))
        for k in rg:
            assert np.array_equal(rg[k][keep].view(np.uint8), ru[k][keep].view(np.uint8)), (b, k)
            for sl, f in fresh.items():
                assert np.array_equal(rg[k][[sl]].view(np.uint8), read(f)[k][[0]].view(np.uint8)), (b, k, sl)


def test_ms_gain_per_unit_equals_reference_pairs():
    """35 M/S pairs, each toggling its S (and once its M) meter between -6 and +14 dB at its own blocks, against 35 Msppmdsp pairs
    driven with set_gain"""
    import torch
    import meters_lv2_b200 as B
    n, blocks = 35, RAGGED
    x = S.white(2 * n, sum(blocks), seed=53) * np.float32(1.5)
    xd = torch.from_numpy(x).cuda()
    g = B.NeedleMeters(n, B.PPM_MS)
    ref = [O.Needle(1, O.PPM_MS) for _ in range(n)]
    rng = np.random.default_rng(17)
    gain = np.full((n, 2), -6.0, np.float32)
    pos = 0
    for b, m in enumerate(blocks):
        for u in range(n):
            if rng.random() < 0.4:
                gain[u, 1] = 14.0 if gain[u, 1] == -6.0 else -6.0
            if b == 6 and u % 5 == 0:
                gain[u, 0] = 14.0
            g.set_gain(float(gain[u, 0]), float(gain[u, 1]), unit=u)
            ref[u].set_gain(float(gain[u, 0]), float(gain[u, 1]))
        g.process(xd[:, pos:pos + m])
        for u, r in enumerate(ref):
            r.process(np.ascontiguousarray(x[2 * u:2 * u + 2, pos:pos + m]))
        pos += m
        got = g.read()
        want = np.concatenate([r.read() for r in ref])
        assert np.array_equal(u32(got), u32(want)), b
        assert np.array_equal(u32(g.state()[:, :3]), u32(np.concatenate([r.peek() for r in ref])[:, :3])), b
    assert len(set(gain[:, 1].tolist())) == 2
