"""CPU: every block entry point of the C ABI (b200m_*_process_* / b200m_*_run_*: plain, _ctl_ and ragged, device and host path)
refuses a NULL handle with B200M_E_INVAL and "NULL" in b200m_last_error(), before it looks at anything else.  Every other argument
is valid, so the handle check is the only one that can fail; none of the calls may touch the GPU or crash."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NFRAM = 64


def _entry_points():
    hdr = open(os.path.join(ROOT, "include", "b200meters.h")).read()
    return {m.group(1): [a.strip() for a in m.group(2).split(",")]
            for m in re.finditer(r"\bint\s+(b200m_[a-z0-9]+_(?:process|run)\w*)\s*\(([^)]*)\)", hdr)}


ENTRY = _entry_points()


def test_every_bank_has_its_block_entry_points():
    banks = {n.split("_")[1] for n in ENTRY}
    assert banks == {"ebu", "tpk", "r128", "dr14", "cor", "ppm", "bim", "sdh", "spec", "pw"}, sorted(banks)
    assert len(ENTRY) >= 38, sorted(ENTRY)
    assert any("_ctl_" in n for n in ENTRY) and any("_ragged_" in n for n in ENTRY)


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_null_handle_is_refused(name):
    import meters_lv2_b200 as B
    L = C.CDLL(B.LIB_PATH)                 # its own function objects: the argtypes set here stay in this test
    buf = np.zeros(1 << 16, np.float32)    # input, lengths, control rows, run flags, `fired`: all valid, never read
    types, vals = [], []
    for i, a in enumerate(ENTRY[name]):
        pname = re.split(r"[\s*]+", a)[-1]
        if i == 0:
            assert "*" in a, a
            types.append(C.c_void_p); vals.append(None)
        elif pname == "stream":
            types.append(C.c_void_p); vals.append(None)
        elif "*" in a:
            types.append(C.c_void_p); vals.append(buf.ctypes.data)
        elif a.startswith("size_t"):
            types.append(C.c_size_t); vals.append(NFRAM)
        elif a.startswith("uint32_t"):
            types.append(C.c_uint32); vals.append(NFRAM if pname == "nfram" else 0)
        elif a.startswith("float"):
            types.append(C.c_float); vals.append(0.0)
        else:
            raise AssertionError("unexpected parameter %r of %s" % (a, name))
    fn = getattr(L, name)
    fn.argtypes, fn.restype = types, C.c_int
    L.b200m_last_error.restype = C.c_char_p
    assert fn(*vals) == -1, name            # B200M_E_INVAL
    assert b"NULL" in L.b200m_last_error(), (name, L.b200m_last_error())
