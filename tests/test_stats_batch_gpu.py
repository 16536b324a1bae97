"""GPU: per-instance control of the bit-meter and SigDistHist banks, and the batched mode of the bitmeter and SigDistHist LV2
plugins built on it (StatsHub, csrc/lv2_stats.cu).

Bank level: every instance of a 37-instance bit-meter bank and a 35-instance SigDistHist bank gets its own START / PAUSE /
RESET / AVERAGE / WINDOWED / CLEAR script; each must read bit for bit what its own reference instance reads, and the bit-meter's
closed flags and published snapshots what a private bank of one driven with the bank-wide API reports.
LV2 level: batched instances (B200M_LV2_BATCH) emit the same control replies as private ones in the same cycle and the same
statistics events one cycle later."""
import ctypes as C
import struct

import numpy as np
import pytest

import _oracle as O
import _signals as S
from test_lv2_ebur128_gpu import ATOM, MTR, cfg, obj, position, sequence, urid
from test_lv2_gon_gpu import RETR, _state_iface
from test_lv2_shim_gpu import Plugin, RefPlugin, descriptors
from test_stats_gpu import BLOCKS, _input

pytestmark = pytest.mark.gpu
CAP = 8192


# ---- bank level ---------------------------------------------------------------------------------------------------------
def _script(n, cmds, nblocks, seed):
    """{instance: {block: [cmd, ...]}}: every command somewhere, plus random ones"""
    rng = np.random.default_rng(seed)
    sc = {i: {} for i in range(n)}
    for i in range(n):
        sc[i].setdefault(2 + (5 * i) % (nblocks - 4), []).append(cmds[i % len(cmds)])
        for b in range(1, nblocks):
            if rng.random() < 0.12:
                sc[i].setdefault(b, []).append(cmds[rng.integers(len(cmds))])
    return sc


class _RefBim:
    """one reference bit-meter instance; RESET = bim_reset, which keeps the window clock: a new reference instance is brought to
    the same clock by replaying the block sizes seen so far while paused (nothing is acquired, so nothing else changes)"""

    def __init__(self, rate):
        self.rate, self.avg, self.integ, self.sizes = rate, False, True, []
        self.o = O.Bitmeter(1, rate)

    def cmd(self, c, B):
        if c == B.CTL_START:
            self.integ = True
        elif c == B.CTL_PAUSE:
            self.integ = False
        elif c == B.CTL_AVERAGE:
            self.avg = True
        elif c == B.CTL_WINDOWED:
            self.avg = False
        elif c == B.CTL_RESET:
            self.o = O.Bitmeter(1, self.rate)
            self.o.mode(self.avg, False)
            for nb in self.sizes:
                self.o.process(np.zeros((1, nb), np.float32))
        elif c == B.CTL_CLEAR:
            self.o, self.avg, self.integ, self.sizes = O.Bitmeter(1, self.rate), False, True, []
        self.o.mode(self.avg, self.integ)

    def process(self, x):
        self.o.process(x)
        self.sizes.append(x.shape[1])


def _published(bank):
    import meters_lv2_b200 as B
    h = np.empty(584, np.int32); c = np.empty(5, np.int32); mm = np.empty(2, np.float32); it = C.c_int64(0)
    B._ck(B.lib().b200m_bim_published(bank.h, 0, B._np_ptr(h), B._np_ptr(c), B._np_ptr(mm), C.byref(it), B._stream_ptr(None)))
    return h, c, mm, it.value


@pytest.mark.parametrize("rate", [48000.0, 44100.0])
def test_bitmeter_per_instance_control(rate):
    import torch
    import meters_lv2_b200 as B
    n = 37
    cmds = [B.CTL_START, B.CTL_PAUSE, B.CTL_RESET, B.CTL_AVERAGE, B.CTL_WINDOWED, B.CTL_CLEAR]
    sc = _script(n, cmds, len(BLOCKS), 41)
    x = _input(n, sum(BLOCKS), 34)
    xd = torch.from_numpy(x).cuda()
    g = B.Bitmeter(n, rate)
    refs = [_RefBim(rate) for _ in range(n)]
    privs = [B.Bitmeter(1, rate) for _ in range(n)]                       # bank of one, bank-wide API
    pos, closes = 0, 0
    for bi, nb in enumerate(BLOCKS):
        for i in range(n):
            for c in sc[i].get(bi, []):
                g.control(c, inst=i); privs[i].control(c); refs[i].cmd(c, B)
        g.run(xd[:, pos:pos + nb])
        for i in range(n):
            privs[i].run(xd[i:i + 1, pos:pos + nb])
            refs[i].process(np.ascontiguousarray(x[i:i + 1, pos:pos + nb]))
        pos += nb
        r = g.results_all()
        for i in range(n):
            oh, oc, om, ot = refs[i].o.read(0)
            assert np.array_equal(r["hist"][i], oh), (bi, i, int((r["hist"][i] != oh).sum()))
            assert np.array_equal(r["cnt"][i], oc) and np.array_equal(r["minmax"][i].view(np.uint32), om.view(np.uint32)) and r["itime"][i] == ot, \
                (bi, i, r["cnt"][i], oc, r["minmax"][i], om, r["itime"][i], ot)
            closed = B.lib().b200m_bim_window_closed(privs[i].h)
            assert r["closed"][i] == closed, (bi, i)
            closes += closed
            ph, pc, pm, pt = _published(privs[i])
            assert np.array_equal(r["pub_hist"][i], ph) and np.array_equal(r["pub_cnt"][i], pc), (bi, i)
            assert np.array_equal(r["pub_minmax"][i].view(np.uint32), pm.view(np.uint32)) and r["pub_itime"][i] == pt, (bi, i)
        # the single-instance readers agree with the bulk read
        h1, c1, m1, t1 = g.results(n - 1)
        assert np.array_equal(h1, r["hist"][n - 1]) and np.array_equal(c1, r["cnt"][n - 1]) and t1 == r["itime"][n - 1]
    assert closes > n * 2


def test_sigdist_per_instance_control():
    import torch
    import meters_lv2_b200 as B
    n = 35
    cmds = [B.CTL_START, B.CTL_PAUSE, B.CTL_RESET, B.CTL_CLEAR]
    sc = _script(n, cmds, len(BLOCKS), 42)
    for i in range(n):
        sc[i].setdefault(0, []).insert(0, B.CTL_START)                    # SigDistHist instances start paused
    x = _input(n, sum(BLOCKS), 35)
    xd = torch.from_numpy(x).cuda()
    g = B.SigDistHist(n)
    refs, integ = [O.SigDist(1) for _ in range(n)], [False] * n
    pos = 0
    for bi, nb in enumerate(BLOCKS):
        for i in range(n):
            for c in sc[i].get(bi, []):
                g.control(c, inst=i)
                if c in (B.CTL_START, B.CTL_PAUSE):
                    integ[i] = c == B.CTL_START
                else:                                                      # RESET: sdh_reset; CLEAR: a new instance
                    refs[i] = O.SigDist(1)
                    integ[i] = integ[i] and c == B.CTL_RESET
                refs[i].integrate(integ[i])
        g.run(xd[:, pos:pos + nb])
        for i in range(n):
            refs[i].process(np.ascontiguousarray(x[i:i + 1, pos:pos + nb]))
        pos += nb
        h, mp, av, it = g.results_all()
        for i in range(n):
            oh, op, oa, ot = refs[i].read(0)
            assert np.array_equal(h[i], oh) and np.array_equal(mp[i], op) and it[i] == ot, (bi, i, it[i], ot)
            assert np.array_equal(av[i].view(np.uint64), oa.view(np.uint64)), (bi, i, av[i], oa)


def test_control_inst_rejects_bad_arguments():
    import meters_lv2_b200 as B
    g = B.Bitmeter(3); s = B.SigDistHist(3)
    for bank in (g, s):
        with pytest.raises(B.B200MError):
            bank.control(B.CTL_START, inst=3)
        with pytest.raises(B.B200MError):
            bank.control(99, inst=0)
    with pytest.raises(B.B200MError):
        s.control(B.CTL_AVERAGE, inst=1)                                   # the SigDistHist has no averaging mode


# ---- LV2 level ----------------------------------------------------------------------------------------------------------
def _split(buf):
    """a notify buffer -> (control replies, statistics events), each the concatenated bytes of its events"""
    ctl = urid(MTR + b"control")
    size = struct.unpack("<I", buf[:4])[0]
    off, end, rep, st = 16, 8 + size, [], []
    while off + 16 <= end:
        sz = struct.unpack("<I", buf[off + 8:off + 12])[0]
        otype = struct.unpack("<I", buf[off + 20:off + 24])[0]
        (rep if otype == ctl else st).append(buf[off:off + 16 + sz])
        off += 16 + (sz + 7) // 8 * 8
    return b"".join(rep), b"".join(st)


class _Host:
    """one plugin instance with its ports; cycle() connects a control sequence and a block and returns the notify bytes"""

    def __init__(self, p):
        self.p, self.note = p, np.zeros(CAP, np.uint8)

    def cycle(self, events, block):
        self.note[:] = 0xA5
        self.note[:8] = np.frombuffer(struct.pack("<II", CAP - 8, 0), np.uint8)
        self.p.port(0, sequence(events)); self.p.port(1, self.note)
        self.p.port(2, block); self.p.port(3, block)
        self.p.run(block.shape[0])
        size = struct.unpack("<I", self.note[:4].tobytes())[0]
        return self.note[:8 + size].tobytes()

    def restore(self, key, value):
        keep = {}

        @RETR
        def retrieve(handle, k, size, typ, flags):
            if k != urid(key):
                return None
            keep["v"] = C.create_string_buffer(struct.pack("<I", value), 4)
            size[0] = 4; typ[0] = urid(ATOM + b"Int"); flags[0] = 3
            return C.addressof(keep["v"])
        _state_iface(self.p if isinstance(self.p, Plugin) else self.p.p).restore(self.p.h, retrieve, None, 0, None)

    def close(self):
        self.p.close()


def _scripts():
    on, off = obj(MTR + b"meteron"), obj(MTR + b"meteroff")
    bim = [{1 + i: [on]} for i in range(6)]
    bim[0].update({20: [cfg("PAUSE", 0)], 35: [cfg("START", 0)]})
    bim[1].update({25: [cfg("RESET", 0)], 26: [cfg("RESET", 0)]})
    bim[2].update({15: [cfg("AVERAGE", 0)], 60: [cfg("WINDOWED", 0)]})
    bim[3].update({30: [off], 45: [on]})
    bim[5].update({10: [cfg("AVERAGE", 0)], 50: [cfg("RESET", 0)], 70: [cfg("PAUSE", 0)], 71: [cfg("WINDOWED", 0)]})
    sdh = [{1 + i: [on], 2 + i: [cfg("START", 0)]} for i in range(6)]
    sdh[0].update({20: [cfg("PAUSE", 0)], 30: [cfg("START", 0)]})
    sdh[1].update({25: [cfg("RESET", 0)]})
    sdh[2].update({10: [cfg("TRANSPORTSYNC", 1.0), cfg("AUTORESET", 1.0), position(0.0)], 20: [position(1.0)], 40: [position(0.0)],
                   50: [position(1.0)]})
    sdh[3].update({30: [off], 45: [on]})
    sdh[5].update({12: [cfg("UISETTINGS", 3.0)], 60: [cfg("PAUSE", 0)], 61: [cfg("RESET", 0)], 70: [cfg("START", 0)]})
    # state restores before a cycle's run(): bitmeter averaging on, SigDistHist ui_settings 3 | transport follow << 8
    restores = {("bitmeter", 4): (40, MTR + b"bim_state", 1), ("SigDistHist", 4): (40, MTR + b"sdh_state", 3 | 1 << 8)}
    return {"bitmeter": bim, "SigDistHist": sdh}, restores


def test_batched_stats_plugins_match_private_instances(monkeypatch):
    """B200M_LV2_BATCH=8: six bitmeter and six SigDistHist instances, each with its own control script.  Control replies equal a
    private instance's in the same cycle; the statistics events of cycle k + 1 equal the private instance's of cycle k."""
    import meters_lv2_b200 as B
    mine, _ = descriptors(B.LIB_PATH)
    names, nb, blk = ("bitmeter", "SigDistHist"), 90, 1024
    monkeypatch.delenv("B200M_LV2_BATCH", raising=False)
    priv = {nm: [_Host(Plugin(mine[nm])) for _ in range(6)] for nm in names}
    monkeypatch.setenv("B200M_LV2_BATCH", "8")
    bat = {nm: [_Host(Plugin(mine[nm])) for _ in range(6)] for nm in names}
    live = O.available("reference")
    refs = {nm: [_Host(RefPlugin(nm)) for _ in range(6)] for nm in names} if live else None
    scripts, restores = _scripts()
    x = S.white(12, nb * blk, seed=71) * np.float32(1.5)
    x[3, 5000:9000] = 0.0; x[7, 100:200] = np.float32(1e-41); x[9, 300] = np.inf
    prev = {(nm, i): None for nm in names for i in range(6)}
    stats_seen = {nm: 0 for nm in names}
    for b in range(nb):
        for k, nm in enumerate(names):
            for i in range(6):
                if (nm, i) in restores and restores[(nm, i)][0] == b:
                    _, key, val = restores[(nm, i)]
                    for hosts in (priv, bat) + ((refs,) if live else ()):
                        hosts[nm][i].restore(key, val)
                ev = scripts[nm][i].get(b, [])
                blocks = np.ascontiguousarray(x[6 * k + i, b * blk:(b + 1) * blk])
                outs = [h[nm][i].cycle(ev, blocks.copy()) for h in ((priv, bat) + ((refs,) if live else ()))]
                (pr, ps), (br, bs) = _split(outs[0]), _split(outs[1])
                if live:
                    assert outs[2] == outs[0], (nm, i, b)
                assert br == pr, (nm, i, b)
                if b == 0:
                    assert bs == b"", (nm, i)                                 # nothing collected yet
                else:
                    assert bs == prev[(nm, i)], (nm, i, b, len(bs), len(prev[(nm, i)]))
                prev[(nm, i)] = ps
                stats_seen[nm] += len(ps) > 0
    assert stats_seen["bitmeter"] > 6 * 5 and stats_seen["SigDistHist"] > 6 * 20, stats_seen
    for hosts in (priv, bat) + ((refs,) if live else ()):
        for nm in names:
            for h in hosts[nm]:
                h.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", ["bitmeter", "SigDistHist"])
def test_batched_stats_plugins_survive_a_host_that_breaks_the_contract(name, monkeypatch):
    """3 members of a 4-slot hub: instance 1 is bypassed for ten cycles, the block size drops for four cycles, instance 0 leaves
    and a new instance takes its slot.  One cycle late, instance 1 emits what a private instance fed silence for the skipped
    cycles emits, and the new tenant what a freshly instantiated private instance emits, window phase included."""
    import meters_lv2_b200 as B
    mine, _ = descriptors(B.LIB_PATH)
    monkeypatch.delenv("B200M_LV2_BATCH", raising=False)
    private = _Host(Plugin(mine[name]))
    monkeypatch.setenv("B200M_LV2_BATCH", "4")
    ps = [_Host(Plugin(mine[name])) for _ in range(3)]
    fresh = tenant = None
    x = S.white(4, 2048 * 60, seed=15)
    opening = [obj(MTR + b"meteron")] + ([cfg("START", 0)] if name == "SigDistHist" else [])
    got, want, got_t, want_t = {}, {}, {}, {}
    for b in range(60):
        n = 1024 if 30 <= b < 34 else 2048
        for i, h in enumerate(ps):
            if h is None or (i == 1 and 10 <= b < 20):
                continue
            out = h.cycle(opening if b == 0 else [], np.ascontiguousarray(x[i, b * 2048:b * 2048 + n]))
            if i == 1:
                got[b] = _split(out)
        if tenant is not None:
            blk = np.ascontiguousarray(x[3, b * 2048:b * 2048 + n])
            first = b == 46
            got_t[b] = _split(tenant.cycle(opening if first else [], blk.copy()))
            want_t[b] = _split(fresh.cycle(opening if first else [], blk.copy()))
        skipped = 10 <= b < 20
        want[b] = _split(private.cycle(opening if b == 0 else [], np.zeros(n, np.float32) if skipped else np.ascontiguousarray(x[1, b * 2048:b * 2048 + n])))
        if b == 45:
            ps[0].close(); ps[0] = None                                      # leaves while the others keep running
            monkeypatch.delenv("B200M_LV2_BATCH", raising=False)
            fresh = _Host(Plugin(mine[name]))
            monkeypatch.setenv("B200M_LV2_BATCH", "4")
            tenant = _Host(Plugin(mine[name]))                               # takes the vacated slot
    for b in got:
        assert got[b][0] == want[b][0], (name, b)                          # control replies: same cycle
    for k in list(range(9)) + list(range(19, 59)):
        assert got[k + 1][1] == want[k][1], (name, k)                      # statistics: one cycle late
    assert sum(len(want[k][1]) > 0 for k in range(60)) > 8
    for k in range(46, 59):
        assert got_t[k][0] == want_t[k][0], (name, k)
        assert got_t[k + 1][1] == want_t[k][1], (name, k)
    assert sum(len(want_t[k][1]) > 0 for k in range(46, 59)) >= 2
    for h in ps[1:] + [private, fresh, tenant]:
        h.close()


@pytest.mark.parametrize("name", ["bitmeter", "SigDistHist"])
def test_batched_launches_do_not_grow_with_members(name, monkeypatch):
    """in cycles without control messages, a hub launches the same kernels per cycle whether it has 2 or 8 members"""
    import meters_lv2_b200 as B
    mine, _ = descriptors(B.LIB_PATH)
    monkeypatch.setenv("B200M_LV2_BATCH", "8")
    x = S.white(8, 1024 * 12, seed=3)
    opening = [obj(MTR + b"meteron")] + ([cfg("START", 0)] if name == "SigDistHist" else [])
    per_cycle = []
    for members in (2, 8):
        hs = [_Host(Plugin(mine[name])) for _ in range(members)]
        for b in range(12):
            if b == 4:
                c0 = B.launch_count()
            for i, h in enumerate(hs):
                h.cycle(opening if b == 0 else [], np.ascontiguousarray(x[i, b * 1024:(b + 1) * 1024]))
        per_cycle.append((B.launch_count() - c0) / 8)
        for h in hs:
            h.close()
    assert per_cycle[0] == per_cycle[1] and per_cycle[0] >= 1, per_cycle
