"""GPU parity of the EBU R128 gated statistics beyond stationary noise.

The device copy of Ebu_r128_hist (csrc/ebu.cu: hist_integrate, hist_calc_integ, hist_calc_range) walks the non-zero
bins with warp ballots in the reference's sequential float order (ebu_r128_proc.cc:82-150).  Stationary input fills a
few neighbouring bins and never lets the relative gates remove content, so this file drives those functions with:

 a. synthetic histograms through b200m_ebu_mix_finish (the whole-mix finish runs the same device functions), against the
    reference's own Ebu_r128_hist::calc_integ / calc_range (oracle hist_calc);
 b. program-like loudness (ramps, 20 dB steps, speech-like bursts between silence and room noise, passages that clamp at
    bin 750, the Tech 3341 tone) on stereo, 5-channel and mono banks, every block against the reference, plus an
    independent float64 BS.1770-4 check of integrated loudness;
 c. per-instance START / PAUSE / RESET scripts, which move the host mirror of each instance's S period (phase_ctl,
    phase_tick) that decides when the gate kernel runs;
 d. the sliced host path of the EBUr128 cycle (b200m_r128_run_host) at bank sizes whose slice bounds fall inside a
    K-weighting warp and a true-peak group, against the device path and the reference plugin, in exact and tolerance mode.
"""
import os

import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
RES = ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated", "integ_thr", "range_min", "range_max", "range_thr")
FS = 48000.0
HAVE_REF = O.available("reference")


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------- synthetic histograms
def _spread(rng, total, bins):
    """`total` points over the given bins, every listed bin non-empty when total allows"""
    bins = np.asarray(bins)
    h = np.zeros(751, np.int64)
    if total == 0:
        return h
    w = rng.random(bins.size) + 0.05
    c = np.floor(w / w.sum() * total).astype(np.int64)
    c[rng.integers(0, bins.size)] += total - c.sum()
    np.add.at(h, bins, c)
    return h


def _cluster(rng, centre, width, total):
    lo, hi = max(0, centre - width), min(750, centre + width)
    return _spread(rng, total, np.arange(lo, hi + 1))


def _one_hist(rng, fam, is_s):
    if fam == "threshold":
        total = int(rng.choice([19, 20, 21]) if is_s else rng.choice([49, 50, 51]))
        return _spread(rng, total, rng.integers(300, 700, size=rng.integers(1, 6)))
    if fam == "single":
        h = np.zeros(751, np.int64)
        h[int(rng.choice([0, 99, 100, 699, 700, 750]))] = int(rng.choice([50, 1000, 77777, 1 << 20]))
        return h
    if fam == "clusters":                       # two groups 15-40 LU apart: the -10 LU / -20 LU gates fall between them
        gap = int(rng.integers(150, 401))
        hi_c = int(rng.integers(gap + 20, 740))
        return _cluster(rng, hi_c, int(rng.integers(0, 20)), int(rng.integers(40, 3000))) + \
            _cluster(rng, hi_c - gap, int(rng.integers(0, 20)), int(rng.integers(40, 3000)))
    if fam == "near0":                          # mean below bin 100: the computed gate bin k is negative and clamps to 0
        return _cluster(rng, int(rng.integers(0, 60)), int(rng.integers(0, 30)), int(rng.integers(60, 5000)))
    if fam == "all":
        return rng.integers(1, 1000, size=751).astype(np.int64)
    if fam == "sparse":
        return _spread(rng, int(rng.integers(60, 100000)), rng.choice(751, size=int(rng.integers(2, 40)), replace=False))
    if fam == "huge":                           # per-bin counts near 2^27: the int -> float conversions round
        nb = int(rng.integers(1, 9))
        h = np.zeros(751, np.int64)
        b = rng.choice(np.arange(200, 751), size=nb, replace=False)
        h[b] = rng.integers(1 << 24, 1 << 27, size=nb) + rng.integers(0, 1 << 10, size=nb)
        return h
    raise ValueError(fam)


FAMILIES = ("threshold", "single", "clusters", "near0", "all", "sparse", "huge")


def hist_families(n_per_family=420, seed=5150):
    """[(family, hist_M int64[751], hist_S int64[751])]: M and S drawn independently from one family"""
    rng = np.random.default_rng(seed)
    out = []
    for fam in FAMILIES:
        for _ in range(n_per_family):
            out.append((fam, _one_hist(rng, fam, False), _one_hist(rng, fam, True)))
    return out


def mix_vector(hm, hs):
    """the b200m_ebu_mix_reduce layout: M bins 0-750, S bins 752-1502, counts at 1504 / 1505, error counts 1506 / 1507"""
    v = np.zeros(1508, np.int64)
    v[:751] = hm; v[752:1503] = hs; v[1504] = hm.sum(); v[1505] = hs.sum()
    assert v.max() < 2 ** 31
    return v.astype(np.int32)


def test_mix_finish_gate_functions_bit_exact():
    """b200m_ebu_mix_finish (hist_calc_integ + hist_calc_range on one warp) on ~3000 synthetic histograms: all five floats
    bit-identical to the reference's Ebu_r128_hist::calc_integ / calc_range, run live (O.hist_calc) and as stored in
    tests/golden/ebu_hist_calc.npz."""
    import torch
    import meters_lv2_b200 as B
    fams = hist_families()
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ebu_hist_calc.npz"))["out5"]
    assert gold.shape == (len(fams), 5)
    mixes = np.stack([mix_vector(hm, hs) for _, hm, hs in fams])
    d = torch.from_numpy(mixes).cuda()
    g = B.Ebu_r128_proc(1, 2)
    gated_i = gated_r = clamped = 0
    for r, (fam, hm, hs) in enumerate(fams):
        got = g.mix_finish(d[r])
        want = O.hist_calc(hm, int(hm.sum()), hs, int(hs.sum()))
        assert np.array_equal(u32(got), u32(want)), (r, fam, got, want, np.nonzero(hm)[0][:8], np.nonzero(hs)[0][:8])
        assert np.array_equal(u32(got), u32(gold[r])), (r, fam, got, gold[r])          # the reference's stored outputs
        # does the family reach the cases it is meant to?  (the relative gates remove occupied bins; k clamps to 0)
        if hm.sum() >= 50:
            k_i = int(np.floor(10.0 * want[1] + 700.5))            # bin of the -10 LU gate
            gated_i += int(np.nonzero(hm)[0].min() < k_i)
            clamped += int(k_i < 0)
        if hs.sum() >= 20:
            gated_r += int(np.nonzero(hs)[0].min() < int(np.floor(10.0 * want[4] + 700.5)))
    assert gated_i > 300 and gated_r > 300 and clamped > 100, (gated_i, gated_r, clamped)


# ---------------------------------------------------------------------------------------------- program-like input
class Program:
    """Program-like input for n_inst instances of nchan channels, generated block by block (counter-based: block b
    of a run depends only on the seed, b and the frames before it).  Each instance follows its own envelope over about
    -80 .. +10 dBFS on uniform noise; instance kind = inst % 4:
      0  slow sine ramps of 30 dB plus 20 dB steps,
      1  speech-like bursts (4 Hz syllable modulation) separated by digital silence or by room noise at -82 dBFS
         (below the -70 LUFS absolute gate),
      2  loud passages at +7 .. +10 dBFS (M and S above +5 LUFS: clamped to bin 750) between quiet ones,
      3  a triangle ramp from -80 to +2 dBFS and back.
    Instance 0 is the EBU Tech 3341 tone: 997 Hz at -23 dBFS on the first two channels (the first, for mono)."""

    def __init__(self, n_inst, nchan, seed):
        self.n, self.nchan, self.seed, self.pos, self.blk = n_inst, nchan, seed, 0, 0
        rng = np.random.default_rng(seed)
        self.kind = np.arange(n_inst) % 4
        self.period = rng.uniform(6.0, 25.0, n_inst)
        self.step = rng.uniform(1.3, 4.0, n_inst)
        self.base = rng.uniform(-55.0, -35.0, n_inst)
        self.phase = rng.uniform(0.0, 2 * np.pi, n_inst)
        self.sched = {}
        for i in range(n_inst):
            if self.kind[i] in (1, 2):
                self.sched[i] = self._schedule(rng, self.kind[i])
        self.chan_db = -1.5 * (np.arange(nchan) % 3)

    @staticmethod
    def _schedule(rng, kind, horizon=400.0):
        """alternating on / off segments: (edges, level dB, off-kind) ; off-kind 0 = digital silence, 1 = room noise"""
        edges, lev, off = [0.0], [], []
        t = 0.0
        while t < horizon:
            on = rng.uniform(0.15, 1.4) if kind == 1 else rng.uniform(1.5, 4.0)
            gap = rng.uniform(0.1, 0.9) if kind == 1 else rng.uniform(1.5, 4.0)
            lev += [rng.uniform(-32.0, -12.0) if kind == 1 else rng.uniform(7.0, 10.0), rng.uniform(-40.0, -30.0)]
            off += [0, int(rng.integers(0, 2)) if kind == 1 else 2]
            t += on; edges.append(t); t += gap; edges.append(t)
        return np.array(edges), np.array(lev), np.array(off)

    def gain(self, t):
        """[n_inst, len(t)] linear gain at times t (seconds)"""
        n = self.n
        g = np.empty((n, t.size), np.float64)
        for kind in range(4):
            idx = np.nonzero(self.kind == kind)[0]
            if kind == 0:
                db = self.base[idx, None] + 15.0 * np.sin(2 * np.pi * t[None, :] / self.period[idx, None] + self.phase[idx, None]) \
                    + 20.0 * (np.floor(t[None, :] / self.step[idx, None]) % 2)
                g[idx] = 10.0 ** (db / 20.0)
            elif kind == 3:
                u = (t[None, :] / (2 * self.period[idx, None]) + self.phase[idx, None] / (2 * np.pi)) % 1.0
                db = -80.0 + 82.0 * (1.0 - np.abs(2.0 * u - 1.0))
                g[idx] = 10.0 ** (db / 20.0)
            else:
                for i in idx:
                    edges, lev, off = self.sched[i]
                    s = np.searchsorted(edges, t, side="right") - 1
                    on = (s % 2) == 0
                    gi = 10.0 ** (lev[s] / 20.0)
                    if kind == 1:
                        gi = np.where(on, gi * (0.2 + 0.8 * np.sin(np.pi * 4.0 * t + i) ** 2),
                                      np.where(off[s] == 1, 10.0 ** (-82.0 / 20.0), 0.0))
                    g[i] = gi
        return g

    CTL = 32                                    # the envelopes are evaluated once per 32 frames and held

    def next(self, nfram):
        frames = self.pos + np.arange(nfram)
        t = frames / FS
        c = frames // self.CTL
        env = self.gain(np.arange(c[0], c[-1] + 1) * (self.CTL / FS))[:, c - c[0]]
        rng = np.random.Generator(np.random.Philox(key=self.seed, counter=[0, 0, self.blk, 0]))
        noise = rng.random((self.n * self.nchan, nfram), dtype=np.float32) * np.float32(2.0) - np.float32(1.0)
        g = np.repeat(env, self.nchan, axis=0) * np.tile(10.0 ** (self.chan_db / 20.0), self.n)[:, None]
        x = noise * g.astype(np.float32)
        tone = (10 ** (-23 / 20) * np.sin(2 * np.pi * 997.0 * t)).astype(np.float32)
        x[:self.nchan] = 0.0
        x[0] = tone
        if self.nchan >= 2:
            x[1] = tone
        self.pos += nfram; self.blk += 1
        return np.ascontiguousarray(x)


def ragged_blocks(seconds, seed):
    """mostly 1024-frame blocks with 1, 7, 2401, 4799 and 8192 mixed in, at least `seconds` of audio"""
    rng = np.random.default_rng(seed)
    out, tot = [], 0
    while tot < seconds * FS:
        n = 1024 if rng.random() < 0.8 else int(rng.choice([1, 7, 2401, 4799, 8192]))
        out.append(n); tot += n
    return out


def oracle_counts(o):
    """[n_inst, 4]: hist_M_count, hist_S_count, error_M, error_S"""
    return np.stack([o.hist(i)[2] for i in range(o.n)])


def _k_weight_loudness_blocks(x):
    """independent float64 BS.1770-4: K-weighting (48 kHz coefficients of the recommendation), mean square per channel
    over 400 ms blocks every 100 ms, loudness -0.691 + 10 log10 (sum of channel mean squares).  A block ending at
    t < 400 ms averages over the 400 ms window with silence before the start, as the meter's zero-initialised ring does."""
    from scipy.signal import lfilter
    b1, a1 = [1.53512485958697, -2.69169618940638, 1.19839281085285], [1.0, -1.69065929318241, 0.73248077421585]
    b2, a2 = [1.0, -2.0, 1.0], [1.0, -1.99004745483398, 0.99007225036621]
    y = lfilter(b2, a2, lfilter(b1, a1, x.astype(np.float64), axis=1), axis=1)
    hop = int(FS) // 10
    nb = y.shape[1] // hop
    e = (y[:, :nb * hop] ** 2).reshape(y.shape[0], nb, hop).sum(axis=2).sum(axis=0)      # energy per 100 ms, channels summed
    ep = np.concatenate([np.zeros(3), e])
    win = (ep[0:nb] + ep[1:nb + 1] + ep[2:nb + 2] + ep[3:nb + 3]) / (4 * hop)          # block j ends with hop j
    return -0.691 + 10 * np.log10(np.maximum(win, 1e-300))


def _gated_integrated(lk):
    """BS.1770-4 gating: absolute -70 LUFS, relative -10 LU below the power mean of the blocks above it"""
    p = 10 ** ((lk + 0.691) / 10)
    a = lk > -70.0
    rel = -0.691 + 10 * np.log10(p[a].mean()) - 10.0
    sel = a & (lk > rel)
    return -0.691 + 10 * np.log10(p[sel].mean())


# The meter's integrated loudness is the power mean of its M points after each is replaced by the centre of its 0.1 LU
# bin (ebu_r128_proc.cc:70,82-101): that moves each point, hence the mean, by at most half a bin, 0.05 LU.  Its block
# loudness uses -0.6976 where BS.1770-4 has -0.691 (0.0066 LU), and its gates act on bins, so a point within half a bin of
# a gate may fall on the other side: each such point changes a power mean over N >= 500 points by at most
# 10 log10 (1 + 1 / N) < 0.009 LU.  Allowing two such points: 0.05 + 0.0066 + 2 * 0.009 < 0.08 LU.
I_FLOAT64_BOUND_LU = 0.08


@pytest.mark.parametrize("n_inst,nchan", [(131, 2), (45, 5), (33, 1)])
def test_program_loudness_bank_vs_reference(n_inst, nchan):
    """131 stereo instances (partial warps in K1 and K2b, a partial K2a CTA), 45 five-channel and 33 mono instances on
    60 s of program-like input in ragged blocks: after every block the nine floats and the histogram point counts of every
    instance equal the reference's bit for bit; at the end every histogram bin, the whole-mix sum and its finish."""
    import torch
    import meters_lv2_b200 as B
    gen = Program(n_inst, nchan, seed=4100 + nchan)
    blocks = ragged_blocks(61.0, seed=nchan)
    g = B.Ebu_r128_proc(n_inst, nchan); o = O.Ebu(n_inst, nchan)
    g.integr_start(); o.integr("start")
    check = [0, 1, 3, 4, 5] if nchan == 2 else []
    keep = []
    for bi, n in enumerate(blocks):
        x = gen.next(n)
        g.process(torch.from_numpy(x).cuda()); o.process(x, nthreads=8)
        gr, orr = g.results(), o.read()
        for i, name in enumerate(RES):
            bad = np.nonzero(u32(gr[name]) != u32(orr[:, i]))[0]
            assert bad.size == 0, (bi, n, name, bad[:5], gr[name][bad[:3]], orr[bad[:3], i])
        oc = oracle_counts(o)
        assert np.array_equal(gr["hist_M_count"], oc[:, 0]) and np.array_equal(gr["hist_S_count"], oc[:, 1]), bi
        if check:
            keep.append(x[[2 * i + c for i in check for c in range(2)]].copy())
    oc = oracle_counts(o)
    assert oc[:, 0].min() >= 300 and oc[:, 1].min() >= 30
    assert (oc[:, 2] > 0).sum() >= n_inst // 5, "the loud instances must reach the bin-750 clamp"
    gr = g.results()
    assert (gr["integrated"] > -100).all() and (gr["range_max"] > -100).all()
    mix_m = np.zeros(751, np.int64); mix_s = np.zeros(751, np.int64); words = np.zeros(4, np.int64)
    for i in range(n_inst):
        hm, hs = g.histogram(i)
        om, os_, c4 = o.hist(i)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_), i
        mix_m += om; mix_s += os_; words += c4
    mix = torch.zeros(B.MIX_WORDS, dtype=torch.int32, device="cuda")
    g.mix_reduce(mix)
    m = mix.cpu().numpy()
    assert np.array_equal(m[:751], mix_m) and np.array_equal(m[752:1503], mix_s) and np.array_equal(m[1504:1508], words)
    assert np.array_equal(u32(g.mix_finish(mix)), u32(O.hist_calc(mix_m, int(words[0]), mix_s, int(words[1]))))
    if check:
        x = np.concatenate(keep, axis=1)
        for j, i in enumerate(check):
            want = _gated_integrated(_k_weight_loudness_blocks(x[2 * j:2 * j + 2]))
            assert abs(float(gr["integrated"][i]) - want) <= I_FLOAT64_BOUND_LU, (i, float(gr["integrated"][i]), want)
        assert abs(float(gr["integrated"][0]) + 23.0) < 0.05                 # Tech 3341 case 1


# ---------------------------------------------------------------------------------------------- gate schedule
def _control_script(n_inst, nblocks, seed):
    """per block: list of (cmd, inst) applied before the block; cmd in start / pause / reset, inst -1 = bank-wide.
    Block 0 starts the whole bank (one S phase for everyone); per-instance controls then spread the instances over the
    ten phases, and an occasional bank-wide control gathers them again."""
    rng = np.random.default_rng(seed)
    script = [[("start", -1)]]
    for b in range(1, nblocks):
        ops = []
        for _ in range(int(rng.poisson(0.25))):
            ops.append((str(rng.choice(["start", "pause", "reset"], p=[0.45, 0.3, 0.25])), int(rng.integers(0, n_inst))))
        if rng.random() < 0.004:
            ops.append((str(rng.choice(["start", "pause", "reset"])), -1))
        script.append(ops)
    return script


@pytest.mark.parametrize("api", ["ebu", "r128"])
def test_gate_schedule_per_instance_controls(api):
    """67 stereo instances, a seeded script of per-instance and bank-wide integr_start / pause / reset landing at every
    phase of the 10-fragment S period: the gate kernel runs only where the host mirror (phase_ctl / phase_tick) predicts a
    wrap, so one missed phase leaves an instance's I / LRA stale.  Nine floats after every block, div1 / div2 at the end.
    `r128` drives the same script through EBUr128.control (START / PAUSE / RESET) on the device path."""
    import torch
    import meters_lv2_b200 as B
    n_inst = 67
    gen = Program(n_inst, 2, seed=6700)
    blocks = ragged_blocks(30.0, seed=67)
    script = _control_script(n_inst, len(blocks), seed=68 if api == "ebu" else 69)
    o = O.Ebu(n_inst, 2)
    if api == "ebu":
        g = B.Ebu_r128_proc(n_inst, 2); ebu = g
        ctl = {"start": g.integr_start, "pause": g.integr_pause, "reset": g.integr_reset}
    else:
        g = B.EBUr128(n_inst, FS, dbtp_enable=True); ebu = g.ebu
        code = {"start": B.EBUr128.START, "pause": B.EBUr128.PAUSE, "reset": B.EBUr128.RESET}
        ctl = {k: (lambda inst, c=c: g.control(c, inst)) for k, c in code.items()}
    phases = {k: set() for k in ("start", "pause", "reset")}
    ran = np.zeros(n_inst, bool)
    for bi, n in enumerate(blocks):
        for cmd, inst in script[bi]:
            for i in (range(n_inst) if inst < 0 else [inst]):
                phases[cmd].add(int(o.state(i)[3][3]))
            ctl[cmd](inst); o.integr(cmd, inst)
        x = gen.next(n)
        xd = torch.from_numpy(x).cuda()
        if api == "ebu":
            g.process(xd)
        else:
            g.run(xd)
        o.process(x, nthreads=8)
        gr, orr = ebu.results(), o.read()
        for i, name in enumerate(RES):
            bad = np.nonzero(u32(gr[name]) != u32(orr[:, i]))[0]
            assert bad.size == 0, (bi, n, name, bad[:5], gr[name][bad[:3]], orr[bad[:3], i])
        ran |= gr["integrated"] > -100
    assert all(p == set(range(10)) for p in phases.values()), phases
    assert ran.sum() >= n_inst // 2
    for i in range(n_inst):
        gc, oc = ebu.state(i)[3], o.state(i)[3]
        assert list(gc) == list(oc), (i, gc, oc)
        hm, hs = ebu.histogram(i); om, os_, _ = o.hist(i)
        assert np.array_equal(hm, om) and np.array_equal(hs, os_), i


# ---------------------------------------------------------------------------------------------- sliced host path
class _Feeds:
    """the same block through the device path (CUDA tensor), a dense pinned host buffer (b200m_host_alloc: one DMA per
    slice when the block fills the staging rows) and a strided numpy view 12 bytes into wider rows (the 2-D copy)"""

    def __init__(self, rows):
        import meters_lv2_b200 as B
        self.B, self.rows, self.pinned = B, rows, {}
        self.wide = np.zeros((rows, 8192 + 8), np.float32)

    def dense(self, x):
        n = x.shape[1]
        if n not in self.pinned:
            self.pinned[n] = self.B.host_alloc(self.rows, n)
        p = self.pinned[n]
        p[:] = x
        return p

    def strided(self, x):
        v = self.wide[:, 3:3 + x.shape[1]]
        v[:] = x
        return v


_REF_CACHE = {}


def _reference_readings(n_inst, seconds, seed):
    """the reference's EBUr128 plugin (ebur128_run) on the Program input: [n_inst, 10] = nine getters + tp_max.
    Without oracle/_ref: the port's restatement of Ebu_r128_proc and TruePeakdsp::process_max, tp_max by numpy log10."""
    key = (n_inst, seconds, seed)
    if key in _REF_CACHE:
        return _REF_CACHE[key]
    gen = Program(n_inst, 2, seed=seed)
    blocks = ragged_blocks(seconds, seed=seed)
    if HAVE_REF:
        p = O.EbuPlugin(n_inst, FS, True)
        for n in blocks:
            p.run(gen.next(n), nthreads=8)
        out = p.read()
    else:
        oe, ot = O.Ebu(n_inst, 2), O.TruePeak(2 * n_inst)
        oe.integr("start")
        tpmax = np.full(n_inst, -np.inf, np.float32)
        for n in blocks:
            x = gen.next(n)
            oe.process(x, nthreads=8); ot.process(x, mode=1, nthreads=8)
            m, _ = ot.read()
            v = np.maximum(m[0::2], m[1::2])
            with np.errstate(divide="ignore"):
                tpmax = np.maximum(tpmax, np.where(v == 0, -np.inf, 20.0 * np.log10(v.astype(np.float64))).astype(np.float32))
        out = np.concatenate([oe.read(), tpmax[:, None]], axis=1)
    _REF_CACHE[key] = out
    return out


SLICED = [(n, s, c) for n in (70, 131) for s in (1, 3, 4, 8) for c in (0, 1, 2)] + \
         [(65, 1, 1), (65, 3, 2), (65, 4, 1), (65, 8, 0), (1000, 3, 2), (1000, 4, 1), (1000, 8, 1)]


@pytest.mark.parametrize("n_inst,slices,concurrent", SLICED)
def test_sliced_host_path_exact(monkeypatch, n_inst, slices, concurrent):
    """b200m_r128_run_host splits the bank into B200M_R128_SLICES slices at n_inst * s / slices: for these sizes the bounds
    fall inside a 32-channel K-weighting warp and an 8-channel true-peak group.  After every block the host banks (dense
    pinned buffer, strided view) equal the device path bit for bit, results and tp_max; at the end all equal the reference
    EBUr128 plugin bit for bit (tp_max within 2 ulp when only the port is available: numpy's log10 is not log10f)."""
    import torch
    import meters_lv2_b200 as B
    monkeypatch.setenv("B200M_R128_SLICES", str(slices))
    monkeypatch.setenv("B200M_R128_CONCURRENT", str(concurrent))
    seconds, seed = 11.0, 7000 + n_inst
    gen = Program(n_inst, 2, seed=seed)
    blocks = ragged_blocks(seconds, seed=seed)
    dev, hd, hs = (B.EBUr128(n_inst, FS, True) for _ in range(3))
    for b in (dev, hd, hs):
        b.control(B.EBUr128.START)
    feeds = _Feeds(2 * n_inst)
    for bi, n in enumerate(blocks):
        x = gen.next(n)
        dev.run(torch.from_numpy(x).cuda())
        hd.run(feeds.dense(x))
        hs.run(feeds.strided(x))
        rd, td = dev.results()
        for what, bank in (("dense", hd), ("strided", hs)):
            rh, th = bank.results()
            assert rh.tobytes() == rd.tobytes(), (what, bi, n)
            assert np.array_equal(u32(th), u32(td)), (what, bi, n)
    ref = _reference_readings(n_inst, seconds, seed)
    res, tp = dev.results()
    for i, name in enumerate(RES):
        bad = np.nonzero(u32(res[name]) != u32(ref[:, i]))[0]
        assert bad.size == 0, (name, bad[:5])
    assert (res["integrated"] > -100).sum() >= n_inst - 2
    if HAVE_REF:
        assert np.array_equal(u32(tp), u32(ref[:, 9])), np.nonzero(u32(tp) != u32(ref[:, 9]))[0][:5]
    else:
        fin = np.isfinite(ref[:, 9])
        assert np.array_equal(np.isfinite(tp), fin)
        assert np.abs(tp[fin].astype(np.float64) - ref[fin, 9].astype(np.float64)).max() <= 8e-6          # 2 ulp at 32 dB
    for i in sorted({0, n_inst // 3, n_inst // 2 + 1, n_inst - 1}):
        a, c = dev.histogram(i), hs.histogram(i)
        assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]), i


def test_sliced_host_path_tolerance_mode():
    """tolerance mode (B200M_PREC_FMA), as bench.py's end-to-end figure runs it: n_inst = 16 n_sm + 5, so that each of the
    4 slices holds at least n_sm 8-channel groups (tpmax_tc_kernel) and slices 1-3 start at channel % 8 = 2, 4, 6.  Blocks
    of 1024 frames alternate with lengths that are not multiples of 4 (tpmax_kernel).  EBU floats and histograms are
    bit-identical to the reference, tp_max within 1e-4 dB of it, and the host path equals the device path bit for bit:
    a channel's arithmetic does not depend on the slice it lands in."""
    import torch
    import meters_lv2_b200 as B
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_inst = 16 * n_sm + 5
    bounds = [2 * (n_inst * s // 4) for s in range(5)]
    assert sorted(b % 8 for b in bounds[1:4]) == [2, 4, 6] and min((bounds[s + 1] - bounds[s]) // 8 for s in range(4)) >= n_sm
    gen = Program(n_inst, 2, seed=8800)
    blocks = []
    while sum(blocks) < 3.0 * FS:
        blocks += [1024] * 6 + [1023, 1024, 2401, 1024, 7]
    dev, host = B.EBUr128(n_inst, FS, True), B.EBUr128(n_inst, FS, True)
    for b in (dev, host):
        b.set_precision(B.PREC_FMA); b.control(B.EBUr128.START)
    oe, ot = O.Ebu(n_inst, 2), O.TruePeak(2 * n_inst)
    oe.integr("start")
    tpmax = np.full(n_inst, -np.inf, np.float32)
    feeds = _Feeds(2 * n_inst)
    for bi, n in enumerate(blocks):
        x = gen.next(n)
        dev.run(torch.from_numpy(x).cuda())
        host.run(feeds.dense(x))
        oe.process(x, nthreads=8); ot.process(x, mode=1, nthreads=8)
        m, _ = ot.read()
        v = np.maximum(m[0::2], m[1::2])
        with np.errstate(divide="ignore"):
            tpmax = np.maximum(tpmax, np.where(v == 0, -np.inf, 20.0 * np.log10(v.astype(np.float64))).astype(np.float32))
        rd, td = dev.results(); rh, th = host.results()
        assert rh.tobytes() == rd.tobytes(), (bi, n)
        bad = np.nonzero(u32(th) != u32(td))[0]
        assert bad.size == 0, (bi, n, bad[:5], th[bad[:3]], td[bad[:3]])
    orr = oe.read()
    for i, name in enumerate(RES):
        assert np.array_equal(u32(rd[name]), u32(orr[:, i])), name
    fin = np.isfinite(tpmax)
    assert np.array_equal(np.isfinite(td), fin)
    assert np.abs(td[fin].astype(np.float64) - tpmax[fin].astype(np.float64)).max() <= 1e-4
    for i in range(0, n_inst, 7):
        hm, hs_ = host.histogram(i); om, os_, _ = oe.hist(i)
        assert np.array_equal(hm, om) and np.array_equal(hs_, os_), i
