"""PCM input without a GPU: the numpy restatement's known answers for every format, the C entry point's argument checks (which
refuse before any device use), and pcm_source's checks of dtype, shape and format when a source is built."""
import ctypes as C

import numpy as np
import pytest

import meters_lv2_b200 as B
import _pcm as P

B200MError = B.B200MError


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_known_answers_s16():
    a = np.array([[[-32768, 32767], [0, -1], [16384, -16384]]], np.int16)
    want = np.array([-1.0, 32767 / 32768, 0.0, -1 / 32768, 0.5, -0.5], np.float32)
    assert np.array_equal(bits(P.values(a, P.S16).ravel()), bits(want))
    assert np.array_equal(P.planar(a, P.S16), want.reshape(3, 2).T)


def test_known_answers_s24():
    def packed(v):
        return np.array([[[[x & 0xff, (x >> 8) & 0xff, (x >> 16) & 0xff] for x in v]]], np.uint8)
    got = P.values(packed([0x800000, 0x7fffff, 0xffffff, 0x000001, 0x400000, 0xc00000]), P.S24).ravel()
    want = np.array([-1.0, (2 ** 23 - 1) / 2 ** 23, -2.0 ** -23, 2.0 ** -23, 0.5, -0.5], np.float32)
    assert np.array_equal(bits(got), bits(want))


def test_known_answers_s32():
    a = np.array([[[-2 ** 31, 2 ** 31 - 1, 0, 1, -1, 2 ** 24 + 1, 2 ** 24 + 3]]], np.int32)
    got = P.values(a, P.S32).ravel()
    # INT32_MAX rounds to 2^31: 1.0; 2^24 + 1 and 2^24 + 3 are ties, rounded to the even 2^24 and 2^24 + 4
    want = np.array([-1.0, 1.0, 0.0, 2.0 ** -31, -2.0 ** -31, 2.0 ** -7, (2 ** 24 + 4) * 2.0 ** -31], np.float32)
    assert np.array_equal(bits(got), bits(want))


def test_known_answers_f32_bit_copy():
    u = np.array([0x7fc00001, 0xffa12345, 0x7f800000, 0xff800000, 0x80000000, 0x00000001, 0x3f800000], np.uint32)
    got = P.values(u.view(np.float32).reshape(1, 1, -1), P.F32).ravel()
    assert np.array_equal(got.view(np.uint32), u)                   # NaN payloads, +-Inf, -0 and denormals kept


def test_planar_layout():
    rng = np.random.default_rng(1)
    a = P.random(rng, 3, 5, 4, P.S16)
    p = P.planar(a, P.S16)
    assert p.shape == (12, 5)
    for i in range(3):
        for c in range(4):
            assert np.array_equal(p[i * 4 + c], a[i, :, c].astype(np.float32) / 32768)


# ---------------------------------------------------------------------------------------------------- C argument checks
def _call(ptr=0x10000, fmt=P.S16, n=2, nchan=2, nfram=16, in_stride=None, out=0x20000, out_stride=64):
    if in_stride is None:
        in_stride = nfram * nchan * P.BYTES[fmt]
    return B.lib().b200m_pcm_planar_device(0, C.c_void_p(ptr), fmt, n, nchan, nfram, in_stride, C.c_void_p(out), out_stride, None)


@pytest.mark.parametrize("kw", [
    dict(ptr=0), dict(out=0), dict(fmt=4, in_stride=128), dict(fmt=-1, in_stride=128), dict(n=0), dict(nchan=0), dict(nchan=33),
    dict(nfram=0), dict(nfram=8193),
    dict(in_stride=63), dict(fmt=P.S24, nchan=2, nfram=16, in_stride=95), dict(ptr=0x10001), dict(fmt=P.S32, ptr=0x10002),
    dict(in_stride=65), dict(fmt=P.F32, in_stride=130), dict(out_stride=15, nfram=16),
], ids=lambda kw: ",".join("%s=%s" % i for i in kw.items()))
def test_c_refuses(kw):
    assert _call(**kw) == -1                                          # B200M_E_INVAL, checked before the device is looked for


def test_c_without_device():
    if B.lib().b200m_device_count() > 0:
        pytest.skip("a CUDA device is present")
    assert _call() == -5                                              # B200M_E_NODEVICE
    assert _call(fmt=P.S24, ptr=0x10001, in_stride=97) == -5        # packed 24-bit: any byte alignment is accepted


# ---------------------------------------------------------------------------------------------------- pcm_source checks
@pytest.fixture
def no_device(monkeypatch):
    """any use of the library (and so of the device) fails the test"""
    def refuse():
        raise AssertionError("pcm_source used the library")
    monkeypatch.setattr(B, "lib", refuse)


@pytest.mark.parametrize("data, kw", [
    (np.zeros((2, 8, 2), np.float64), {}),
    (np.zeros((2, 8, 2), np.int8), {}),
    (np.zeros((2, 8, 2), np.uint8), {}),
    (np.zeros((2, 8, 2, 4), np.uint8), {}),
    (np.zeros((16, 2), np.int16), {}),
    (np.zeros((2, 8, 2, 1), np.int16), {}),
    (np.zeros((0, 8, 2), np.int16), {}),
    (np.zeros((2, 8, 0), np.int16), {}),
    (np.zeros((2, 8, 33), np.int16), {}),
    (np.zeros((2, 8, 2), np.int16), dict(fmt=B.PCM_S32)),
    (np.zeros((2, 8, 2), np.int32), dict(fmt=B.PCM_F32)),
    (np.zeros((2, 8, 2, 3), np.uint8), dict(fmt=B.PCM_S16)),
    (np.zeros((2, 8, 2), np.int16), dict(nchan=1)),
    (lambda off, n: None, {}),
    (lambda off, n: None, dict(nchan=2)),
    (lambda off, n: None, dict(fmt=B.PCM_S16)),
    (lambda off, n: None, dict(nchan=2, fmt=7)),
    (lambda off, n: None, dict(nchan=0, fmt=B.PCM_S16)),
    (lambda off, n: None, dict(nchan=33, fmt=B.PCM_S16)),
    ([[[0, 0]]], {}),
])
def test_pcm_source_refuses(no_device, data, kw):
    with pytest.raises(B200MError):
        B.pcm_source(data, **kw)


def test_pcm_source_accepts(no_device):
    for a, fmt in ((np.zeros((2, 8, 2), np.int16), B.PCM_S16), (np.zeros((2, 8, 6, 3), np.uint8), B.PCM_S24),
                   (np.zeros((1, 8, 32), np.int32), B.PCM_S32), (np.zeros((3, 8, 1), np.float32), B.PCM_F32)):
        assert callable(B.pcm_source(a))
        assert callable(B.pcm_source(a, nchan=a.shape[2], fmt=fmt))
    assert callable(B.pcm_source(lambda off, n: None, nchan=2, fmt=B.PCM_S24))


def test_pcm_source_block_past_end(no_device):
    f = B.pcm_source(np.zeros((2, 100, 2), np.int16))
    for off, n in ((64, 64), (100, 1), (-1, 4), (0, 101), (0, 0), (0, 8193)):
        with pytest.raises(B200MError):
            f(off, n)
