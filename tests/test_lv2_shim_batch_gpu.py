"""GPU: batched mode (B200M_LV2_BATCH) of the control-port plugins with per-instance controls, slot reuse, BBCM6 and the surround
meters.  A batched instance's control ports after cycle k + 1 must equal, bit for bit, those of a private instance after cycle k
(one declared cycle of latency), and the reference plugin's where oracle/_ref is built.  A private instance is a bank of its own,
pinned to the reference by tests/test_lv2_shim_gpu.py."""
import numpy as np
import pytest

import _oracle as O
import _signals as S
from test_lv2_shim_gpu import Plugin, RefPlugin, descriptors

pytestmark = pytest.mark.gpu
BLK = 1024


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def layout(name):
    """(control ports, input control ports, audio (in, out) port pairs, initial control values)"""
    if name.startswith("spectr30"):
        nch = 2 if name.endswith("stereo") else 1
        return list(range(64)), {60, 61, 62, 63}, [(64, 65), (66, 67)][:nch], {60: 1.0, 61: -4.0, 62: 0.0}
    if name.startswith("surround"):
        chn = int(name[8:]); cors = 4 if chn > 3 else 3
        ctl = [0] + [1 + 3 * c + k for c in range(cors) for k in range(3)] + [p for c in range(chn) for p in (15 + 4 * c, 16 + 4 * c)]
        sel = {1 + 3 * c for c in range(cors)} | {2 + 3 * c for c in range(cors)}
        return ctl, {0} | sel, [(13 + 4 * c, 14 + 4 * c) for c in range(chn)], {1 + 3 * c: float(c) for c in range(cors)} | {2 + 3 * c: float(c + 1) for c in range(cors)}
    stereo = not name.endswith("mono")
    km = name[0] == "K" or name.startswith("dBTP")
    ctl = {"COR": [0, 3], "VUstereo": [0, 3, 6], "DINmono": [0, 3], "dBTPstereo": [0, 3, 6, 7, 8], "K20stereo": [0, 3, 6, 7, 8, 9],
           "BBCM6": [0, 3, 6, 7]}[name]
    return ctl, {0, 7} if name == "BBCM6" else {0}, [(1, 2), (4, 5)] if stereo else [(1, 2)], {0: 20.0 if km else -18.0}


class Host:
    """one plugin instance with its control ports; cycle() runs it on one block and returns its output control ports"""

    def __init__(self, plugin, name):
        self.p, self.name = plugin, name
        ctl, self.inputs, self.audio, init = layout(name)
        self.ctl = {i: np.zeros(1, np.float32) for i in ctl}
        for i, v in init.items():
            self.ctl[i][0] = v
        for i, a in self.ctl.items():
            plugin.port(i, a)
        self.outs = [i for i in ctl if i not in self.inputs]

    def cycle(self, bufs, ctl=None):
        for i, v in (ctl or {}).items():
            self.ctl[i][0] = v
        mine = [np.ascontiguousarray(b).copy() for b in bufs]
        for c, (pi, po) in enumerate(self.audio):
            self.p.port(pi, mine[c]); self.p.port(po, mine[c])
        self.p.run(len(mine[0]))
        return {i: np.float32(self.ctl[i][0]) for i in self.outs}

    def close(self):
        self.p.close()


def same(name, got, want, where):
    for i, r in want.items():
        a = got[i]
        if name.startswith("spectr30") and i >= 30 and r <= -500:
            assert a <= -500, (where, i, a, r)                     # rand()-based "force redraw" values (src/spectrumlv2.c:243-246)
        else:
            assert u32(a)[()] == u32(r)[()], (where, i, a, r)


def hosts(name, n, batch, monkeypatch):
    import meters_lv2_b200 as B
    mine, _ = descriptors(B.LIB_PATH)
    if batch:
        monkeypatch.setenv("B200M_LV2_BATCH", str(batch))
    else:
        monkeypatch.delenv("B200M_LV2_BATCH", raising=False)
    return [Host(Plugin(mine[name]), name) for _ in range(n)]


def refs(name, n):
    return [Host(RefPlugin(name), name) for _ in range(n)] if O.available("reference") else []


def run_members(name, n, nb, scripts, x, monkeypatch, nch):
    """n batched members of one hub against n private instances (and reference plugins) fed the same audio and control scripts"""
    bat = hosts(name, n, 8, monkeypatch)
    priv = hosts(name, n, 0, monkeypatch)
    ref = refs(name, n)
    prev = [None] * n
    checked = 0
    for b in range(nb):
        for k in range(n):
            bufs = [x[nch * k + c, b * BLK:(b + 1) * BLK] for c in range(nch)]
            ctl = scripts[k].get(b, {})
            got = bat[k].cycle(bufs, ctl)
            want = priv[k].cycle(bufs, ctl)
            if ref:
                same(name, want, ref[k].cycle(bufs, ctl), ("private vs reference", b, k))
            if prev[k] is not None:
                same(name, got, prev[k], (name, b, k))
                checked += 1
            prev[k] = want
    for h in bat + priv + ref:
        h.close()
    return checked


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", ["spectr30mono", "spectr30stereo"])
def test_batched_spectr30_with_per_instance_speed_and_reset(name, monkeypatch):
    nch = 2 if name.endswith("stereo") else 1
    n, nb = 5, 24
    x = S.white(nch * n, BLK * nb, seed=61)
    scripts = [{3: {60: 3.0}, 9: {61: 1.0}, 10: {61: 3.0}, 12: {61: -3.0}},
               {5: {60: 0.004}, 6: {61: 0.0}, 15: {60: 22.0}},
               {},
               {2: {61: 3.0}, 3: {61: 3.0}, 4: {61: -4.0}, 8: {60: 7.5, 61: -1.0}, 18: {61: 1.0}},
               {1: {60: 15.0}, 11: {61: -3.0}, 13: {61: 0.0}, 20: {60: 1.0}}]
    assert run_members(name, n, nb, scripts, x, monkeypatch, nch) == n * (nb - 1)


@pytest.mark.timeout(300)
def test_batched_bbcm6_with_per_instance_s_gain(monkeypatch):
    n, nb = 5, 20
    x = S.white(2 * n, BLK * nb, seed=63) * np.float32(2.0)
    scripts = [{3: {7: 1.0}, 9: {7: 0.0}}, {}, {5: {7: 1.0}}, {1: {7: 1.0}, 2: {7: 0.0}, 3: {7: 1.0}, 14: {7: 0.0}}, {12: {7: 0.7}}]
    assert run_members("BBCM6", n, nb, scripts, x, monkeypatch, 2) == n * (nb - 1)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("chn", [3, 5, 8])
def test_batched_surround_with_per_instance_pairs(chn, monkeypatch):
    n, nb = 3, 20
    x = S.white(chn * n, BLK * nb, seed=65 + chn)
    for k in range(n):
        x[chn * k + 1] = 0.6 * x[chn * k] + 0.4 * x[chn * k + 1]; x[chn * k + 2] = -x[chn * k]
    cors = 4 if chn > 3 else 3

    def pairs(a, b):
        return {p: float(v) for c in range(cors) for p, v in ((1 + 3 * c, a(c)), (2 + 3 * c, b(c)))}
    scripts = [{0: pairs(lambda c: c, lambda c: (c + 1) % chn)},
               {0: {1: 9.0, 2: 0.0, 4: 2.0, 5: 1.0}, 8: {1: 0.0, 2: 2.0}},                # 9 clamps to chn - 1
               {0: pairs(lambda c: chn - 1 - c, lambda c: 1), 6: {4: 0.0, 5: 1.0}, 13: {7: 40.0}}]
    assert run_members("surround%d" % chn, n, nb, scripts, x, monkeypatch, chn) == n * (nb - 1)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", ["COR", "VUstereo", "DINmono", "spectr30stereo", "dBTPstereo", "K20stereo", "BBCM6", "surround5"])
def test_a_new_tenant_starts_fresh(name, monkeypatch):
    """4 members fill a 4-slot hub; member 0 leaves before cycle 20, its slot idles on silence for five cycles, and a new instance
    takes it at cycle 25.  One cycle late, the tenant reads what a freshly instantiated private instance (and reference plugin) fed its
    audio reads."""
    ctl, _, audio, _ = layout(name)
    nch = len(audio)
    nb = 40
    x = S.white(5 * nch, BLK * nb, seed=67) * np.float32(1.5)
    ctls = {3: {61: 1.0}, 6: {60: 3.0}} if name.startswith("spectr30") else {}     # the first tenant leaves non-default controls
    if name == "BBCM6":
        ctls = {4: {7: 1.0}}
    members = hosts(name, 4, 4, monkeypatch)
    tenant = fresh = None
    ref = []
    got, want = {}, {}
    for b in range(nb):
        for k, h in enumerate(members):
            if h is not None:
                h.cycle([x[nch * k + c, b * BLK:(b + 1) * BLK] for c in range(nch)], ctls.get(b) if k == 0 else None)
        if b == 19:
            members[0].close(); members[0] = None
        if b == 24:
            tenant = hosts(name, 1, 4, monkeypatch)[0]
            fresh = hosts(name, 1, 0, monkeypatch)[0]
            ref = refs(name, 1)
        if b >= 25:
            bufs = [x[nch * 4 + c, b * BLK:(b + 1) * BLK] for c in range(nch)]
            got[b] = tenant.cycle(bufs)
            want[b] = fresh.cycle(bufs)
            if ref:
                same(name, want[b], ref[0].cycle(bufs), ("private vs reference", b))
    for b in range(25, nb - 1):
        same(name, got[b + 1], want[b], (name, b))
    for h in [m for m in members if m is not None] + [tenant, fresh] + ref:
        h.close()


@pytest.mark.parametrize("name", ["spectr30stereo", "BBCM6", "surround5"])
def test_batched_launches_do_not_grow_with_members(name, monkeypatch):
    """in cycles without control changes, a hub launches the same kernels per cycle whether it has 2 or 8 members"""
    import meters_lv2_b200 as B
    _, _, audio, _ = layout(name)
    nch = len(audio)
    x = S.white(8 * nch, BLK * 12, seed=3)
    per_cycle = []
    for members in (2, 8):
        hs = hosts(name, members, 8, monkeypatch)
        for b in range(12):
            if b == 4:
                c0 = B.launch_count()
            for i, h in enumerate(hs):
                h.cycle([x[nch * i + c, b * BLK:(b + 1) * BLK] for c in range(nch)])
        per_cycle.append((B.launch_count() - c0) / 8)
        for h in hs:
            h.close()
    assert per_cycle[0] == per_cycle[1], per_cycle
    assert 1 <= per_cycle[0] <= 4, per_cycle
