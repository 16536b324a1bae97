"""GPU: the goniometer plugin of the LV2 façade (csrc/lv2_gon.cu) side by side with the reference's (src/goniometerlv2.c:44-330,
compiled unmodified into oracle/_ref).  The reference GUI reaches the plugin through LV2 instance-access: it casts the instance
handle to `LV2gm*` (src/goniometer.h:113-169) and reads the ring buffer / flips `ui_active` in it.  The test does exactly that to
BOTH handles, at the offsets the two libraries report for their own structs (which must agree)."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import _oracle as O
import _signals as S
from test_lv2_shim_gpu import Plugin, _map, _uris, descriptors, reference_names, u32

pytestmark = pytest.mark.gpu
FIELDS = ("rb", "ui_active", "rb_overrun", "s_sfact", "s_linewidth", "input", "rate", "ntfy", "msg_thread_lock", "map", "sizeof")
# what the reference's goniometer does in these tests, stored by tests/golden/make_golden.py for machines without oracle/_ref
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "goniometer_ref.npz")


def _layout(lib, fn):
    a = (C.c_size_t * 16)()
    n = getattr(lib, fn)(a, 16)
    return dict(zip(FIELDS, list(a)[:n]))


def _layouts():
    import meters_lv2_b200 as B
    mine = _layout(C.CDLL(B.LIB_PATH), "b200m_lv2_gon_layout")
    if O.available("reference"):
        return mine, _layout(C.CDLL(O.PATHS["reference"]), "refgon_layout")
    return mine, dict(zip(FIELDS, (int(v) for v in np.load(GOLD)["layout"])))


class Ring(C.Structure):                                   # gmringbuf, src/goniometer.h:33-39
    _fields_ = [("c0", C.POINTER(C.c_float)), ("c1", C.POINTER(C.c_float)), ("rp", C.c_size_t), ("wp", C.c_size_t), ("len", C.c_size_t)]


def _ring(handle, off):
    return C.cast(C.c_void_p.from_address(handle + off["rb"]).value, C.POINTER(Ring)).contents


def feed(p, off):
    """24 cycles of the goniometer with a GUI that opens at cycle 4 and drains the ring at cycle 12, through instance-access.
    Returns [25, 6]: (ring length, write pointer) before the first cycle, then after every cycle the correlation and
    notification ports (as bits), the ring's write / read pointers, rb_overrun and ntfy; and digests of the ring's two channels."""
    n, nb = 1024, 24
    x = S.white(2, n * nb, seed=71); x[1, : n * 6] = x[0, : n * 6]
    p.gain = np.ones(1, np.float32); p.corr = np.full(1, 9.0, np.float32); p.ntf = np.full(1, -1.0, np.float32)
    p.port(4, p.gain); p.port(5, p.corr); p.port(6, p.ntf)
    rb = _ring(p.h, off)
    obs = [(rb.len, rb.wp, 0, 0, 0, 0)]
    for b in range(nb):
        if b == 4:                                          # the GUI opens: ui_active = true through instance-access
            C.c_bool.from_address(p.h + off["ui_active"]).value = True
        if b == 12:                                         # the GUI drains the ring (gmrb_read_clear) and acknowledges the overrun
            rb.rp = rb.wp
            C.c_bool.from_address(p.h + off["rb_overrun"]).value = False
        ins = [np.ascontiguousarray(x[c, b * n:(b + 1) * n]) for c in range(2)]
        outs = [np.zeros(n, np.float32) for _ in range(2)]
        p.port(0, ins[0]); p.port(1, outs[0]); p.port(2, ins[1]); p.port(3, outs[1])
        p.run(n)
        assert np.array_equal(outs[0], ins[0]) and np.array_equal(outs[1], ins[1])
        obs.append((int(u32(p.corr)[0]), int(u32(p.ntf)[0]), rb.wp, rb.rp, int(C.c_bool.from_address(p.h + off["rb_overrun"]).value),
                    C.c_uint32.from_address(p.h + off["ntfy"]).value))
    rings = [hashlib.sha256(np.ctypeslib.as_array(getattr(rb, ch), shape=(rb.len,))[:rb.wp].tobytes()).hexdigest() for ch in ("c0", "c1")]
    return np.array(obs, np.int64), rings


def reference_feed():
    if O.available("reference"):
        ref, l2 = descriptors(O.PATHS["reference"])
        r = Plugin(ref["goniometer"])
        out = feed(r, _layout(l2, "refgon_layout"))
        r.close()
        return out
    g = np.load(GOLD)
    return g["feed"], [str(v) for v in g["feed_rings"]]


def test_instance_struct_layout_matches_the_reference():
    mine, ref = _layouts()
    assert mine == ref and mine["sizeof"] == 208


def test_goniometer_feed_and_correlation():
    import meters_lv2_b200 as B
    off, _ = _layouts()
    mine, l1 = descriptors(B.LIB_PATH)
    assert "goniometer" in mine and len(mine) == 38 == len(reference_names())
    g = Plugin(mine["goniometer"])
    got, got_rings = feed(g, off)
    want, want_rings = reference_feed()
    assert tuple(got[0, :2]) == tuple(want[0, :2]) == (9600, 0)
    for b in range(1, len(want)):
        # correlation untouched (9.0) while the GUI is closed, cor->read () after; notification; ring pointers; overrun; ntfy
        assert tuple(got[b]) == tuple(want[b]), (b - 1, got[b], want[b])
    assert got_rings == want_rings
    assert g.corr[0] != 9.0 and abs(g.corr[0]) <= 1.0
    g.close()


STORE = C.CFUNCTYPE(C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32)
RETR = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_size_t), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32))


class Iface(C.Structure):
    _fields_ = [("save", C.CFUNCTYPE(C.c_uint32, C.c_void_p, STORE, C.c_void_p, C.c_uint32, C.c_void_p)),
                ("restore", C.CFUNCTYPE(C.c_uint32, C.c_void_p, RETR, C.c_void_p, C.c_uint32, C.c_void_p))]


def _state_iface(p):
    ext = C.CFUNCTYPE(C.c_void_p, C.c_char_p)(p.d.extension_data)(b"http://lv2plug.in/ns/ext/state#interface")
    return C.cast(ext, C.POINTER(Iface)).contents


def saved_state(p, off):
    """what save() of a goniometer with non-default GUI settings stores: {key URI: (value, type URI, flags)}"""
    C.c_int.from_address(p.h + off["s_sfact"]).value = 8
    C.c_float.from_address(p.h + off["s_linewidth"]).value = 1.25
    C.c_bool.from_address(p.h + off["rb_overrun"] + 1).value = True           # s_autogain follows rb_overrun
    got = {}

    @STORE
    def store(handle, key, value, size, typ, flags):
        got[_uris[key]] = (C.string_at(value, size), _uris[typ], flags)
        return 0
    _state_iface(p).save(p.h, store, None, 0, None)
    return got


def reference_saved_state():
    if O.available("reference"):
        ref, l2 = descriptors(O.PATHS["reference"])
        r = Plugin(ref["goniometer"])
        out = saved_state(r, _layout(l2, "refgon_layout"))
        r.close()
        return out
    g = np.load(GOLD)
    return {bytes(k): (g["state_value_%d" % i].tobytes(), bytes(t), int(f))
            for i, (k, t, f) in enumerate(zip(g["state_keys"], g["state_types"], g["state_flags"]))}


def test_goniometer_state_save_restore():
    """LV2 state (src/goniometerlv2.c:209-294): two atom:Vector blobs; what one plugin saves the other restores identically"""
    import meters_lv2_b200 as B
    off, _ = _layouts()
    mine, l1 = descriptors(B.LIB_PATH)
    p = Plugin(mine["goniometer"])
    ours = saved_state(p, off)
    p.close()
    ref = reference_saved_state()
    assert ours == ref and len(ours) == 2
    # restore the reference's blobs into a fresh instance of ours
    p = Plugin(mine["goniometer"])
    keep = {}

    @RETR
    def retrieve(handle, key, size, typ, flags):
        uri = _uris[key]
        if uri not in ref:
            return None
        data, t, f = ref[uri]
        keep[uri] = C.create_string_buffer(data, len(data))
        size[0] = len(data); typ[0] = _map(None, t); flags[0] = f
        return C.addressof(keep[uri])
    _state_iface(p).restore(p.h, retrieve, None, 0, None)
    assert C.c_int.from_address(p.h + off["s_sfact"]).value == 8
    assert C.c_float.from_address(p.h + off["s_linewidth"]).value == 1.25
    assert C.c_bool.from_address(p.h + off["rb_overrun"] + 1).value is True
    p.close()
