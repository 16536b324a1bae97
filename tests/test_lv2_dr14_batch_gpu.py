"""GPU: batched dr14mono / dr14stereo / TPnRMSmono / TPnRMSstereo (B200M_LV2_BATCH, csrc/lv2_dr14.cu DrHub).  Members of one hub
run their own scripts (follow transport on / off, transport start / stop, dr14reset, the reset button, meteron / meteroff); after
batched cycle k + 1 every output port must be bit-identical to a private instance's after cycle k, and to the reference plugin's
where oracle/_ref is built.  The rand()-based block count of a GUI re-init cycle is compared by regime.  A member that leaves is
replaced mid-run: the newcomer reads, one cycle late, what a freshly instantiated private plugin reads."""
import numpy as np
import pytest

import _oracle as O
from test_dr14_gpu import OUT_MONO, OUT_ST, _connect, _music
from test_lv2_ebur128_gpu import MTR, obj, position, sequence
from test_lv2_shim_gpu import Plugin, descriptors, u32

pytestmark = pytest.mark.gpu
RATE, BLK, NCYC, NMEM = 8000.0, 1024, 130, 6                 # a 3 s window every ~23 cycles


def _script(m):
    """member m's events {cycle: dict(atoms=[...], follow=f, reset=r)}: every member differs"""
    rng = np.random.default_rng(100 + m)
    s = {}
    for c in rng.choice(np.arange(3, NCYC - 2), 5, replace=False):
        kind = int(rng.integers(0, 4))
        ev = s.setdefault(int(c), {"atoms": []})
        if kind == 0:
            ev["reset"] = 1.0
        elif kind == 1:
            ev["atoms"].append(obj(MTR + b"dr14reset"))
        elif kind == 2:
            ev["atoms"] += [position(0.0)]
            s.setdefault(int(c) + 1, {"atoms": []})["atoms"].append(position(1.0))   # transport start: a reset when following
        else:
            ev["atoms"].append(obj(MTR + b"meteron"))
            s.setdefault(int(c) + 2, {"atoms": []})["atoms"].append(obj(MTR + b"meteroff"))
    s.setdefault(1, {"atoms": []})["follow"] = float(m % 2)      # odd members follow the host transport
    return s


class _Member:
    def __init__(self, d, name, nch, script, x):
        self.p, self.nch, self.script, self.x, self.k = Plugin(d[name], RATE), nch, script, x, 0
        ports = OUT_ST if nch == 2 else OUT_MONO
        self.out = {i: np.zeros(1, np.float32) for i in ports}
        self.ctrl = [np.ones(1, np.float32), np.zeros(1, np.float32)]
        self.hist = []

    def run(self, n=BLK):
        ev = self.script.get(self.k, {})
        ctl = sequence(ev.get("atoms", []))
        self.ctrl[0][0] = ev.get("follow", self.ctrl[0][0]); self.ctrl[1][0] = ev.get("reset", 0.0)
        bufs = [np.ascontiguousarray(self.x[c, self.k * BLK:self.k * BLK + n]) for c in range(self.nch)]
        _connect(self.p, self.nch, ctl, self.ctrl, bufs, self.out)
        self.p.run(n)
        self.hist.append({i: np.float32(a[0]) for i, a in self.out.items()})
        self.k += 1

    def close(self):
        self.p.close()


def _same(got, want, what):
    for i, v in want.items():
        if i == 3 and v < 0:                                    # -1 - (rand () & 0xffff): GUI re-init cycle, regime only
            assert got[i] < 0, (what, i)
        else:
            assert u32(np.float32(got[i]))[()] == u32(np.float32(v))[()], (what, i, got[i], v)


@pytest.mark.parametrize("name", ["dr14stereo", "dr14mono", "TPnRMSstereo", "TPnRMSmono"])
def test_batched_members_read_private_cycle_one_late(name, monkeypatch):
    import meters_lv2_b200 as B
    nch = 2 if "stereo" in name else 1
    mine, _ = descriptors(B.LIB_PATH)
    ref = descriptors(O.PATHS["reference"])[0] if O.available("reference") else None
    xs = [_music(nch, (NCYC + 1) * BLK, 20 + m, 0.9 - 0.1 * m) for m in range(NMEM + 1)]
    xs[2][:] = 0.0                                              # a silent member
    scripts = [_script(m) for m in range(NMEM + 1)]
    monkeypatch.delenv("B200M_LV2_BATCH", raising=False)
    priv = [_Member(mine, name, nch, scripts[m], xs[m]) for m in range(NMEM)]
    refs = [_Member(ref, name, nch, scripts[m], xs[m]) for m in range(NMEM)] if ref else []
    monkeypatch.setenv("B200M_LV2_BATCH", "8")
    bat = [_Member(mine, name, nch, scripts[m], xs[m]) for m in range(NMEM)]
    LEAVE = 70
    for k in range(NCYC):
        if k == LEAVE:                                          # member 4 leaves, a new instance takes its slot
            for g in (bat, priv, refs):
                if g:
                    g[4].close()
            bat[4] = _Member(mine, name, nch, scripts[NMEM], xs[NMEM])
            monkeypatch.delenv("B200M_LV2_BATCH")
            priv[4] = _Member(mine, name, nch, scripts[NMEM], xs[NMEM])
            if ref:
                refs[4] = _Member(ref, name, nch, scripts[NMEM], xs[NMEM])
            monkeypatch.setenv("B200M_LV2_BATCH", "8")
        for g in (bat, priv, refs):
            for p in g:
                p.run()
    for m in range(NMEM):
        got, want = bat[m].hist, priv[m].hist
        assert len(got) == len(want)
        for j in range(1, len(got)):                             # batched run j publishes cycle j - 1
            _same(got[j], want[j - 1], (name, m, j, "private"))
            if ref:
                _same(got[j], refs[m].hist[j - 1], (name, m, j, "reference"))
    if nch == 2 and name.startswith("dr14"):
        assert any(1.0 <= h[18] <= 20.0 for p in priv for h in p.hist)      # DR scores became valid: windows were scored
    for g in (bat, priv, refs):
        for p in g:
            p.close()


@pytest.mark.parametrize("name", ["dr14stereo", "TPnRMSmono"])
def test_broken_host_contract_does_not_hang(name, monkeypatch):
    """a member that runs twice in one cycle and a change of n_samples close the open cycle early (INTEGRATION.md §2b)"""
    import meters_lv2_b200 as B
    nch = 2 if "stereo" in name else 1
    mine, _ = descriptors(B.LIB_PATH)
    monkeypatch.setenv("B200M_LV2_BATCH", "4")
    xs = [_music(nch, 40 * BLK, 40 + m, 0.5) for m in range(3)]
    ps = [_Member(mine, name, nch, {}, xs[m]) for m in range(3)]
    for k in range(30):
        for m, p in enumerate(ps):
            if k == 10 and m == 0:
                p.run(); p.k -= 1                               # twice in one cycle
            p.run(512 if 15 <= k < 18 else BLK)                 # n_samples changes for three cycles
    for p in ps:
        assert all(np.isfinite(v) for v in p.hist[-1].values())
        p.close()
