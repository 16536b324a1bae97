"""GPU: batched EBUr128 (B200M_LV2_BATCH, csrc/lv2_ebur128.cu EbuHub) against reference plugins instantiated in the same cycles.

Members join a running hub at different cycles -- before and after a 50 ms fragment edge -- one leaves and a newcomer takes its
slot, and each sends its own START / PAUSE / RESET.  A newcomer's 50 ms fragment clock starts with its own first run(), as a
freshly instantiated plugin's does, so after batched cycle k + 1 every member's ebulevels (M, S, their maxima, integrated
loudness, loudness range and the dBTP hold) equal, bit for bit, the reference plugin's after cycle k.  The histograms enter
through the integrated loudness and the range; tests/test_ebu_phase_gpu.py pins them bin for bin."""
import struct

import numpy as np
import pytest

import _signals as S
from test_lv2_ebur128_gpu import CAP, MTR, _levels, cfg, obj, sequence, urid
from test_lv2_shim_gpu import Plugin, RefPlugin, descriptors

pytestmark = pytest.mark.gpu
NCYC = 360
KEYS = (b"ebu_loudnessM", b"ebu_maxloudnM", b"ebu_loudnessS", b"ebu_maxloudnS", b"ebu_integrated", b"ebu_range_min",
        b"ebu_range_max", b"truepeak")


def _audio(m, n):
    """member m's program: noise and a tone under a level that moves every ~0.3 s (loudness spreads over many bins)"""
    x = S.white(2, n, seed=300 + m) * np.float32(2.0)
    t = np.arange(n) / 48000.0
    x += (0.3 * np.sin(2 * np.pi * (150.0 + 40 * m) * t)).astype(np.float32)
    env = (10.0 ** (-1.5 * (0.5 + 0.5 * np.sin(2 * np.pi * t / (2.1 + 0.3 * m) + m)))).astype(np.float32)
    return np.ascontiguousarray(x * env, np.float32)


class _Member:
    def __init__(self, p, x, first, script, blk):
        self.p, self.x, self.first, self.script, self.blk = p, x, first, script, blk
        self.note = np.zeros(CAP, np.uint8)
        self.levels = []                                  # per run: {key: 4 bytes} of the ebulevels object, or None

    def run(self, k):
        j = k - self.first                                # the member's own cycle count
        ev = self.script.get(j, [])
        self.note[:] = 0
        self.note[:8] = np.frombuffer(struct.pack("<II", CAP - 8, 0), np.uint8)
        bufs = [np.ascontiguousarray(self.x[c, j * self.blk:(j + 1) * self.blk]) for c in range(2)]
        self.p.port(0, sequence(ev)); self.p.port(1, self.note)
        for c in range(2):
            self.p.port(2 + 2 * c, bufs[c]); self.p.port(3 + 2 * c, bufs[c])
        self.p.run(self.blk)
        self.levels.append(_levels(self.note.tobytes()))


def _script(m):
    """meteron, the member's dBTP setting and START in its first cycle, then a PAUSE / START pair, a RESET and a dBTP off / on
    (on / off / on for members that start with it off) of its own"""
    rng = np.random.default_rng(500 + m)
    dbtp = m % 3 != 1
    s = {0: [obj(MTR + b"meteron"), cfg("UISETTINGS", 8 + 64 if dbtp else 8), cfg("START", 0)]}
    a, b, c, d, e, f = sorted(int(v) for v in rng.choice(np.arange(5, 90), 6, replace=False))
    s[a] = [cfg("PAUSE", 0)]; s[b] = [cfg("START", 0)]; s[c] = [cfg("RESET", 0)]
    for k, on in ((d, not dbtp), (e, dbtp), (f, not dbtp) if not dbtp else (f, True)):
        s.setdefault(k, []).append(cfg("UISETTINGS", 8 + 64 if on else 8))
    return s


@pytest.mark.parametrize("blk", [1024, 1000])
def test_late_joiners_read_the_reference_one_cycle_late(blk, monkeypatch):
    """joins at cycles 0, 0, 1, 2, 3, 7, 40 and 117 (the bank's fragment edges fall every 2400 frames, so the joiners' first
    frames lie at different positions inside a fragment); member 1 leaves at cycle 150 and a newcomer takes its slot in the same
    cycle.  Members 1, 4 and 7 start with dBTP off, the others enable it in their first cycle; every member switches it off and
    on again (or on, off and on) mid-run, while others keep theirs on"""
    import meters_lv2_b200 as B
    mine, _ = descriptors(B.LIB_PATH)
    monkeypatch.setenv("B200M_LV2_BATCH", "8")
    joins = {0: [0, 1], 1: [2], 2: [3], 3: [4], 7: [5], 40: [6], 117: [7], 150: [8]}
    LEAVER, LEAVE = 1, 150
    bat, ref = {}, {}
    xs = {m: _audio(m, (NCYC + 1) * blk) for m in range(9)}
    for k in range(NCYC):
        if k == LEAVE:
            bat[LEAVER].p.close(); ref[LEAVER].p.close()
            bat[LEAVER].gone = ref[LEAVER].gone = True
        for m in joins.get(k, []):
            bat[m] = _Member(Plugin(mine["EBUr128"]), xs[m], k, _script(m), blk)
            ref[m] = _Member(RefPlugin("EBUr128"), xs[m], k, _script(m), blk)
        for g in (bat, ref):
            for mem in g.values():
                if not getattr(mem, "gone", False):
                    mem.run(k)
    ids = [urid(MTR + key) for key in KEYS]
    for m in bat:
        got, want = bat[m].levels, ref[m].levels
        assert len(got) == len(want) and len(got) > 30
        checked = 0
        for j in range(1, len(got)):                       # batched run j publishes the member's cycle j - 1
            for key, name in zip(ids, KEYS):
                assert got[j][key] == want[j - 1][key], (blk, m, j, name, struct.unpack("<f", got[j][key]),
                                                         struct.unpack("<f", want[j - 1][key]))
            checked += 1
        assert checked == len(got) - 1
    assert struct.unpack("<f", bat[5].levels[-1][ids[4]])[0] > -200      # a late joiner's integrated loudness is live
    for g in (bat, ref):
        for m, mem in g.items():
            if not getattr(mem, "gone", False):
                mem.p.close()
