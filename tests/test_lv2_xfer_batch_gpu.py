"""GPU: batched mode (B200M_LV2_BATCH) of the phasewheel and goniometer plugins, which share the COR plugin's correlation hub of
their sample rate.  With COR, phasewheel and goniometer instances mixed in 8-slot hubs, a batched instance's phase / correlation
port after run k + 1 must equal, bit for bit, a private instance's after run k; everything the host sees in the cycle itself --
notify buffers, the goniometer's ring buffer, its pointers, rb_overrun and ntfy -- must be identical in the same cycle.  A
phasewheel cycle whose notify buffer is too small is skipped without metering (held in the bank), a member leaves and another
joins its slot, and the stereoscope (no bank) stays byte-identical.  Where oracle/_ref is built the private instances are also
compared with the reference plugins."""
import ctypes as C
import hashlib
import struct

import numpy as np
import pytest

import _oracle as O
import _signals as S
from test_lv2_ebur128_gpu import MTR, obj, sequence
from test_lv2_gon_gpu import _layouts, _ring
from test_lv2_shim_gpu import Plugin, descriptors, u32

pytestmark = pytest.mark.gpu
BLK, NB = 1024, 24
CAP, SMALL = 16384, 8000                                   # a rawstereo message of 1024 frames needs 8448 bytes (src/xfer.c:188-205)
DELAYED = {"COR": "lvl", "phasewheel": "phase", "goniometer": "corr", "stereoscope": None}
INIT = {"lvl": 7.0, "phase": 5.0, "corr": 9.0}


class Member:
    """one plugin instance with its ports; cycle() runs one block under the instance's script and returns what it published"""

    def __init__(self, plugin, name, script, off, ours=True):
        self.p, self.name, self.script, self.off, self.ours = plugin, name, script, off, ours
        self.ctl = {k: np.full(1, v, np.float32) for k, v in INIT.items()}
        if name == "COR":                                      # src/meters.cc:59-70
            self.refl = np.full(1, -18.0, np.float32)
            plugin.port(0, self.refl); plugin.port(3, self.ctl["lvl"])
            self.audio = [(1, 2), (4, 5)]
        elif name == "goniometer":                             # src/goniometerlv2.c:27-35
            self.gain, self.ntf = np.ones(1, np.float32), np.full(1, -1.0, np.float32)
            plugin.port(4, self.gain); plugin.port(5, self.ctl["corr"]); plugin.port(6, self.ntf)
            self.audio = [(0, 1), (2, 3)]
            self.rb, self.wrapped = _ring(plugin.h, off), False
        else:                                                  # src/xfer.c:50-60
            self.note = np.zeros(CAP, np.uint8)
            plugin.port(1, self.note); plugin.port(6, self.ctl["phase"])
            self.audio = [(2, 3), (4, 5)]

    def flag(self, field):
        return C.c_bool.from_address(self.p.h + self.off[field])

    def cycle(self, b, bufs):
        ev = self.script.get(b, {})
        outs = [np.zeros(BLK, np.float32) for _ in bufs]
        for (pi, po), i, o in zip(self.audio, bufs, outs):
            self.p.port(pi, i); self.p.port(po, o)
        got = {}
        if self.name in ("phasewheel", "stereoscope"):
            cap = SMALL if ev.get("small") else CAP
            self.note[:] = 0xA5
            self.note[:8] = np.frombuffer(struct.pack("<II", cap - 8, 0), np.uint8)
            self.p.port(0, sequence([obj(MTR + m) for m in ev.get("msgs", [])]))
        if self.name == "goniometer":
            if "ui" in ev:                                     # the GUI opens / closes through instance-access
                self.flag("ui_active").value = ev["ui"]
            if ev.get("drain"):                                # gmrb_read_clear, and the GUI acknowledges the overrun
                self.rb.rp = self.rb.wp
                self.flag("rb_overrun").value = False
        wp = self.rb.wp if self.name == "goniometer" else 0
        self.p.run(BLK)
        for i, o in zip(bufs, outs):                           # the reference drops the audio of a skipped xfer cycle (src/xfer.c:190-205)
            assert np.array_equal(i, o) or not self.ours, (self.name, b)
        if self.name in ("phasewheel", "stereoscope"):
            got["note"] = self.note.tobytes()
        if self.name == "goniometer":
            self.wrapped |= self.rb.wp < wp
            hi = self.rb.len if self.wrapped else self.rb.wp
            ring = b"".join(np.ctypeslib.as_array(getattr(self.rb, ch), shape=(self.rb.len,))[:hi].tobytes() for ch in ("c0", "c1"))
            got.update(ntf=int(u32(self.ntf)[0]), wp=self.rb.wp, rp=self.rb.rp, ovr=bool(self.flag("rb_overrun").value),
                       ntfy=C.c_uint32.from_address(self.p.h + self.off["ntfy"]).value, ring=hashlib.sha256(ring).hexdigest())
        if DELAYED[self.name]:
            got[DELAYED[self.name]] = int(u32(self.ctl[DELAYED[self.name]])[0])
        return got

    def close(self):
        self.p.close()


def bits(v):
    return int(u32(np.float32(v))[0])


def script(name, i):
    s = {}
    if name in ("phasewheel", "stereoscope"):
        for b, m in ((2 + i, b"ui_on"), (4 + i, b"ui_on"), (13, b"ui_off"), (15 + i % 2, b"ui_on")):
            s.setdefault(b, {}).setdefault("msgs", []).append(m)
        # too small for this cycle's rawstereo: the cycle is skipped, metering and messages included (the ui_on of cycle 2 + i)
        for b in (2 + i, 5, 6, 11 + i % 3, 18, 22):
            s.setdefault(b, {})["small"] = True
    elif name == "goniometer":
        for b, ev in ((1 + i, {"ui": True}), (7, {"drain": True}), (9 + i % 2, {"ui": False}), (12, {"ui": True}), (16, {"drain": True}),
                      (20 + i % 3, {"ui": False})):
            s.setdefault(b, {}).update(ev)
    return s


def check(name, got, want, where):
    """a batched instance's cycle against its private twin's: same-cycle observables now, the delayed port one cycle late"""
    b, first = where[1], where[2]
    key = DELAYED[name]
    for k, v in want[b].items():
        if k != key:
            assert got[b][k] == v, (where, k)
    if key and b > first:
        assert got[b][key] == want[b - 1][key], (where, key, got[b][key], want[b - 1][key])
    if key and b == first and name != "COR":
        assert got[b][key] == bits(INIT[key]), (where, key)     # nothing published before a first cycle


def against_reference(name, mine, ref, where):
    for k, v in ref.items():
        if k == "note":                                        # our sequence (the reference leaves the rest of the buffer as it found it)
            size = struct.unpack("<I", mine[k][:4])[0]
            n = 8 + size if size < CAP - 8 else CAP
            assert mine[k][:n] == v[:n], where
        else:
            assert mine[k] == v, (where, k)


@pytest.mark.timeout(600)
def test_batched_phasewheel_goniometer_and_cor_share_one_correlation_hub(monkeypatch):
    import meters_lv2_b200 as B
    mine, _ = descriptors(B.LIB_PATH)
    off, _ = _layouts()
    live_ref = O.available("reference")
    ref_desc = descriptors(O.PATHS["reference"])[0] if live_ref else None
    names = [("phasewheel", "goniometer", "COR")[k % 3] for k in range(16)] + ["stereoscope"]   # two full 8-slot hubs
    per = {}
    scripts = []
    for nm in names:
        scripts.append(script(nm, per.get(nm, 0))); per[nm] = per.get(nm, 0) + 1

    def make(nm, sc, batch):
        if batch:
            monkeypatch.setenv("B200M_LV2_BATCH", "8")
        else:
            monkeypatch.delenv("B200M_LV2_BATCH", raising=False)
        return Member(Plugin(mine[nm]), nm, sc, off)

    bat = [make(nm, sc, True) for nm, sc in zip(names, scripts)]
    priv = [make(nm, sc, False) for nm, sc in zip(names, scripts)]
    ref = [Member(Plugin(ref_desc[nm]), nm, sc, off, ours=False) for nm, sc in zip(names, scripts)] if live_ref else []
    first = [0] * len(names)
    x = S.white(2 * (len(names) + 1), BLK * NB, seed=97)
    for k in range(len(names) + 1):
        x[2 * k + 1] = np.float32(0.6) * x[2 * k] + np.float32(0.4) * x[2 * k + 1]
    hist_b = [dict() for _ in names]
    hist_p = [dict() for _ in names]
    leaver, joiner = 3, len(names)                             # a phasewheel of the first hub leaves; a goniometer takes its slot
    for b in range(NB):
        if b == 10:
            for grp in (bat, priv, ref):
                if grp:
                    grp[leaver].close(); grp[leaver] = None
        if b == 12:
            names.append("goniometer"); sc = script("goniometer", 7)
            bat.append(make("goniometer", sc, True)); priv.append(make("goniometer", sc, False))
            if live_ref:
                ref.append(Member(Plugin(ref_desc["goniometer"]), "goniometer", sc, off, ours=False))
            first.append(b); hist_b.append({}); hist_p.append({})
        for k, nm in enumerate(names):
            if bat[k] is None:
                continue
            col = joiner if k == joiner else k
            bufs = [np.ascontiguousarray(x[2 * col + c, b * BLK:(b + 1) * BLK]) for c in range(2)]
            hist_b[k][b] = bat[k].cycle(b, bufs)
            hist_p[k][b] = priv[k].cycle(b, bufs)
            if ref:
                against_reference(nm, hist_p[k][b], ref[k].cycle(b, bufs), ("private vs reference", nm, b, k))
            check(nm, hist_b[k], hist_p[k], (nm, b, first[k], k))
    # the script skipped metering cycles and moved both correlation ports
    assert any(bytes(h[b]["note"][:8]) == struct.pack("<II", SMALL - 8, 0) for h in hist_p[:1] for b in h)
    assert hist_p[0][NB - 1]["phase"] != bits(INIT["phase"])
    assert hist_p[joiner][NB - 1]["corr"] != bits(INIT["corr"])
    for grp in (bat, priv, ref):
        for m in grp:
            if m is not None:
                m.close()
