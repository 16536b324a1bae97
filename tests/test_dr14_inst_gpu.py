"""GPU: per-instance reset_peaks and clear in the DR-14 bank (b200m_dr14_control, csrc/dr14.cu).  Every instance of a shared
bank has its own 3 s window phase, so a bank whose instances are reset and cleared on scripts of their own must read, field for
field and bin for bin, what one bank of one per instance reads when driven with b200m_dr14_reset (a clear: a new bank of one).
Where oracle/_ref is built the reference dr14stereo / dr14mono plugins run alongside, reset through their reset button."""
import numpy as np
import pytest

import _oracle as O
from test_dr14_gpu import OUT_MONO, OUT_ST, _connect, _music
from test_lv2_ebur128_gpu import sequence
from test_lv2_shim_gpu import Plugin, descriptors, u32

pytestmark = pytest.mark.gpu
RATE = 8000.0                                   # the lowest common rate: a window (24001 samples) every ~12 blocks
W = int(np.rint(np.float32(RATE * 3.0))) + 1
FIELDS = ("v_rms", "v_peak", "m_peak", "m_rms", "dr", "dr_total", "block_count")


def _blocks(n, seed):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, 4097, n)
    sizes[[3, 40, 41, 90]] = 1
    sizes[[10, 11, 60, 120]] = 8192
    return sizes


def _script(ninst, sizes, seed):
    """{block: [(inst, cmd), ...]}: random resets and clears, resets in consecutive blocks, resets in the very block where the
    instance's window would close, and never-touched instances 0 and 1"""
    import meters_lv2_b200 as B
    rng = np.random.default_rng(seed)
    script = {}
    for i in range(2, ninst):
        for b in rng.choice(len(sizes), 3, replace=False):
            script.setdefault(int(b), []).append((i, B.DR14_CLEAR if rng.random() < 0.3 else B.DR14_RESET))
    for b in (30, 31, 32):
        script.setdefault(b, []).append((2, B.DR14_RESET))
    # instances whose window closes in block b (phases mirrored here) are reset right there, before the block runs
    phase, t = np.zeros(ninst, np.int64), 0
    for b, n in enumerate(sizes):
        ev = script.get(b, [])
        if b == len(sizes) // 2:
            phase[:] = t % W
        for i, _ in ev:
            phase[i] = t % W
        closing = [i for i in range(2, ninst) if (phase[i] + W - 1 - t % W) % W < n]
        if b in (25, 70, 71, 130) and closing:
            i = closing[b % len(closing)]
            script.setdefault(b, []).append((i, B.DR14_RESET))
            phase[i] = t % W
        t += int(n)
    return script


class _Ref:
    """the reference plugin per instance (oracle/_ref), reset with its reset button, cleared by a new instance"""

    def __init__(self, ninst, nch):
        d, _ = descriptors(O.PATHS["reference"])
        self.d, self.nch, self.name = d, nch, "dr14stereo" if nch == 2 else "dr14mono"
        self.p = [Plugin(d[self.name], RATE) for _ in range(ninst)]
        self.ports = OUT_ST if nch == 2 else OUT_MONO
        self.out = [{k: np.zeros(1, np.float32) for k in self.ports} for _ in range(ninst)]
        self.ctl = sequence([])

    def clear(self, i):
        self.p[i].close()
        self.p[i] = Plugin(self.d[self.name], RATE)

    def run(self, i, x, reset):
        c = [np.ones(1, np.float32), np.full(1, 1.0 if reset else 0.0, np.float32)]
        _connect(self.p[i], self.nch, self.ctl, c, [np.ascontiguousarray(x[k]) for k in range(self.nch)], self.out[i])
        self.p[i].run(x.shape[1])
        o = self.out[i]
        r = dict(v_peak=[o[6][0]], m_peak=[o[7][0]], v_rms=[o[8][0]], m_rms=[o[9][0]], dr=[o[10][0]], block_count=o[3][0])
        if self.nch == 2:
            for k, p in (("v_peak", 13), ("m_peak", 14), ("v_rms", 15), ("m_rms", 16), ("dr", 17)):
                r[k].append(o[p][0])
            r["dr_total"] = o[18][0]
        return r

    def close(self):
        for p in self.p:
            p.close()


def _run(nch, ninst, seed, monkeypatch, env, reference):
    import torch
    import meters_lv2_b200 as B
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sizes = _blocks(160, seed)
    total = int(sizes.sum())
    gains = np.linspace(0.9, 0.05, ninst).astype(np.float32)
    x = np.concatenate([_music(nch, total, seed + i, gains[i]) for i in range(ninst)], axis=0)
    silent, nan_inst = ninst - 1, ninst - 2
    x[silent * nch:(silent + 1) * nch] = 0.0                   # a silent instance: never scored
    x[nan_inst * nch, total // 3] = np.nan                      # a NaN poisons one window of this instance
    xd = torch.from_numpy(x).cuda()
    script = _script(ninst, sizes, seed)
    bank = B.DR14(ninst, nch, RATE, True)
    one = [B.DR14(1, nch, RATE, True) for _ in range(ninst)]
    ref = _Ref(ninst, nch) if reference else None
    t, prev, scored = 0, np.zeros(ninst, np.float32), set()
    for b, n in enumerate(sizes):
        n = int(n)
        ev = script.get(b, [])
        pressed = set()
        if b == len(sizes) // 2:                                 # a bank-wide reset in the middle
            bank.reset()
            for s in one:
                s.reset()
            pressed = set(range(ninst))
        resets = [i for i, c in ev if c == B.DR14_RESET]
        clears = [i for i, c in ev if c == B.DR14_CLEAR]
        if resets:
            bank.control(B.DR14_RESET, resets)                  # one call per block for every listed instance
        if clears:
            bank.control(B.DR14_CLEAR, clears)
        for i in resets:
            one[i].reset(); pressed.add(i)
        for i in clears:
            one[i] = B.DR14(1, nch, RATE, True)
            if ref:
                ref.clear(i)
        bank.run(xd[:, t:t + n])
        got = bank.results()
        if (got["block_count"] > prev).any():
            scored.add(b)
        prev = got["block_count"].copy()
        for i in range(ninst):
            one[i].run(xd[i * nch:(i + 1) * nch, t:t + n])
            want = one[i].results()
            for k in FIELDS:
                assert np.array_equal(u32(got[k][i]), u32(want[k][0])), (b, i, k, got[k][i], want[k][0])
            if ref:
                r = ref.run(i, x[i * nch:(i + 1) * nch, t:t + n], i in pressed)
                for k, v in r.items():
                    a = np.atleast_1d(got[k][i])[:nch] if k not in ("dr_total", "block_count") else got[k][i:i + 1]
                    assert np.array_equal(u32(a), u32(np.atleast_1d(np.float32(v)))), ("reference", b, i, k, a, v)
        t += n
    res = bank.results()
    for i in range(ninst):
        for c in range(nch):
            assert np.array_equal(bank.histogram(i, c), one[i].histogram(0, c)), (i, c)
    assert res["block_count"][silent] == 0.0
    assert len(scored) >= 25, sorted(scored)                    # staggered phases: windows close in many different blocks
    if ref:
        ref.close()
    return script


FORMS = {"fused": {}, "wide": {"B200M_TPK_WIDE": "2", "B200M_TPK_SPLIT": "0"},
         "slabs": {"B200M_TPK_SPLIT": "2", "B200M_TPK_SLAB": "192"}}


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("nch,ninst", [(2, 24), (1, 20)])
def test_dr14_per_instance_reset_and_clear(form, nch, ninst, monkeypatch):
    reference = O.available("reference")
    script = _run(nch, ninst, 11 + nch, monkeypatch, FORMS[form], reference)
    touched = {i for ev in script.values() for i, _ in ev}
    assert 0 not in touched and 1 not in touched and len(touched) == ninst - 2


def test_dr14_control_arguments():
    import meters_lv2_b200 as B
    bank = B.DR14(4, 2, RATE, True)
    with pytest.raises(Exception):
        bank.control(B.DR14_RESET, [4])
    with pytest.raises(Exception):
        bank.control(7, [0])
    bank.control(B.DR14_RESET, [])                              # an empty list does nothing
    bank.control(B.DR14_CLEAR, [1, 1, 3])                       # repeats are one reset
    bank.control(B.DR14_CLEAR)
