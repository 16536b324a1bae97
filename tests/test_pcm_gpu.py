"""PCM input on the device: b200m_pcm_planar_device against the numpy restatement (tests/_pcm.py) bit for bit, and every programme_*
function fed pcm_source against the same function fed the restatement's float32 planar host array, in exact mode."""
import ctypes as C

import numpy as np
import pytest
import torch

import meters_lv2_b200 as B
import _pcm as P

pytestmark = pytest.mark.gpu

FORMATS = (P.S16, P.S24, P.S32, P.F32)
MAX_SAMPLES = 1 << 24          # N * nchan * nfram per case: N = 4096 with the wider blocks would take gigabytes


def u32(t):
    return np.ascontiguousarray(t.cpu().numpy() if torch.is_tensor(t) else t, np.float32).view(np.uint32)


def upload(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("nfram", [1, 3, 4, 1023, 1024, 8192])
@pytest.mark.parametrize("nchan", [1, 2, 3, 6, 12, 32])
@pytest.mark.parametrize("fmt", FORMATS)
def test_kernel_bitexact(fmt, nchan, nfram):
    rng = np.random.default_rng(1000 * fmt + 10 * nchan + nfram)
    for n in (1, 7, 4096):
        if n * nchan * nfram > MAX_SAMPLES:
            continue
        a = P.random(rng, n, nfram, nchan, fmt)
        out = B.pcm_planar(upload(a), fmt, nchan)
        assert out.shape == (n * nchan, nfram) and out.stride(0) % 64 == 0
        assert np.array_equal(u32(out), u32(P.planar(a, fmt))), (n, nchan, nfram)


def _raw_call(d_in, fmt, n, nchan, nfram, in_stride, d_out, out_stride, stream=None):
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream if stream is None else stream.cuda_stream)
    return B.lib().b200m_pcm_planar_device(0, C.c_void_p(d_in), fmt, n, nchan, nfram, in_stride, C.c_void_p(d_out), out_stride, st)


SENTINEL = 0x7fbadbad          # a NaN pattern in out's padding, which no call may write


@pytest.mark.parametrize("fmt", FORMATS)
def test_strides_and_offsets(fmt):
    """clips at every allowed byte offset from a 16-byte boundary, padded in_stride and out_stride: the rows match, the padding of
    out keeps its sentinel"""
    rng = np.random.default_rng(7 + fmt)
    align = 1 if fmt == P.S24 else P.BYTES[fmt]
    n, nchan, nfram = 7, 3, 1023
    clip = nfram * nchan * P.BYTES[fmt]
    for off in range(0, 16, align):
        for pad in (0, align, 16 + align, 64):
            in_stride = clip + pad
            a = P.random(rng, n, nfram, nchan, fmt)
            buf = rng.integers(0, 256, size=off + n * in_stride + 32, dtype=np.uint8)
            rows = buf[off:off + n * in_stride].reshape(n, in_stride)
            rows[:, :clip] = P.raw(a, fmt)
            d_in = upload(buf)
            out_stride = nfram + 5
            d_out = torch.full((n * nchan, out_stride), SENTINEL, dtype=torch.int32, device="cuda")
            assert _raw_call(d_in.data_ptr() + off, fmt, n, nchan, nfram, in_stride, d_out.data_ptr(), out_stride) == 0
            got = d_out.cpu().numpy().view(np.uint32)
            assert np.array_equal(got[:, :nfram], u32(P.planar(a, fmt))), (off, pad)
            assert (got[:, nfram:] == SENTINEL).all()


def test_non_default_stream_and_launches():
    rng = np.random.default_rng(3)
    a = P.random(rng, 64, 1024, 2, P.S16)
    d = upload(a)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    before = B.launch_count()
    out = B.pcm_planar(d, P.S16, 2, stream=s)
    assert B.launch_count() - before == 1                                   # one launch per call
    s.synchronize()
    assert np.array_equal(u32(out), u32(P.planar(a, P.S16)))
    with torch.cuda.stream(s):                                              # torch's current stream
        before = B.launch_count()
        out = B.pcm_planar(d, P.S16, 2, nfram=1000)
        assert B.launch_count() - before == 1
    s.synchronize()
    assert np.array_equal(u32(out), u32(P.planar(a[:, :1000], P.S16)))


def test_refused_arguments_leave_out_untouched():
    n, nchan, nfram = 4, 2, 64
    d_in = torch.zeros(n * nfram * nchan * 4 + 64, dtype=torch.uint8, device="cuda")
    d_out = torch.full((n * nchan, nfram), SENTINEL, dtype=torch.int32, device="cuda")
    p, o = d_in.data_ptr(), d_out.data_ptr()
    good = dict(d_in=p, fmt=P.S16, n=n, nchan=nchan, nfram=nfram, in_stride=nfram * nchan * 2, d_out=o, out_stride=nfram)
    bad = [dict(d_in=0), dict(d_out=0), dict(fmt=4), dict(fmt=-1), dict(n=0), dict(nchan=0), dict(nchan=33), dict(nfram=0),
           dict(nfram=8193, out_stride=8193), dict(in_stride=nfram * nchan * 2 - 2), dict(d_in=p + 1), dict(in_stride=nfram * nchan * 2 + 1),
           dict(fmt=P.S32, in_stride=nfram * nchan * 4 + 2), dict(fmt=P.S32, d_in=p + 2, in_stride=nfram * nchan * 4),
           dict(fmt=P.F32, in_stride=nfram * nchan * 4 - 4), dict(fmt=P.S24, in_stride=nfram * nchan * 3 - 1), dict(out_stride=nfram - 1)]
    before = B.launch_count()
    for kw in bad:
        assert _raw_call(**{**good, **kw}) == -1, kw
    torch.cuda.synchronize()
    assert B.launch_count() == before
    assert (d_out.cpu().numpy().view(np.uint32) == SENTINEL).all()


# ---------------------------------------------------------------------------------------------------- programme functions
def same(a, b, path="out"):
    """a == b field by field, arrays compared byte for byte (NaN-aware: equal NaN bit patterns match)"""
    if isinstance(a, dict):
        assert isinstance(b, dict) and sorted(a) == sorted(b), path
        for k in a:
            same(a[k], b[k], "%s[%r]" % (path, k))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), path
        for k, (x, y) in enumerate(zip(a, b)):
            same(x, y, "%s[%d]" % (path, k))
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape, path
        assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes(), path


def clips(rng, fmt, n, t, nchan):
    """n clips of audio-like PCM (noise and a sine at per-clip levels, a few clipped samples): [n, t, nchan(, 3)]"""
    lvl = 10.0 ** (-rng.uniform(0, 30, size=(n, 1, 1)) / 20)
    f = rng.uniform(50, 5000, size=(n, 1, 1))
    x = lvl * (0.5 * np.sin(2 * np.pi * f * np.arange(t)[None, :, None] / 48000 + rng.uniform(0, 6, size=(1, 1, nchan)))
               + 0.5 * rng.uniform(-1, 1, size=(n, t, nchan)))
    x[:, ::997] *= 4.0                                                       # overs and clipped samples
    if fmt == P.F32:
        return x.astype(np.float32)
    top = 2.0 ** (8 * P.BYTES[fmt] - 1)
    v = np.clip(np.round(x * top), -top, top - 1).astype(np.int64)
    if fmt == P.S24:
        u = (v & 0xffffff).astype(np.uint32)
        return np.stack([u & 0xff, (u >> 8) & 0xff, (u >> 16) & 0xff], axis=-1).astype(np.uint8)
    return v.astype(P.DTYPE[fmt])


N_CLIPS, T_MAX, BLOCK = 12, 3 * 48000 + 4321, 1000          # past one 3 s DR window; every clip ends inside a block


@pytest.fixture(scope="module")
def s16():
    rng = np.random.default_rng(11)
    a = clips(rng, P.S16, N_CLIPS, T_MAX, 2)
    lengths = rng.integers(1, T_MAX, size=N_CLIPS)
    lengths[0] = T_MAX
    lengths[1] = 3 * BLOCK + 7
    lengths[lengths % BLOCK == 0] += 1
    return a, lengths, np.ascontiguousarray(P.planar(a, P.S16))


GROUPS = np.where(np.arange(N_CLIPS) == 5, -1, np.arange(N_CLIPS) % 3)     # three albums and one clip in none


@pytest.mark.parametrize("name, fn", [
    ("loudness", lambda x, ln: B.programme_loudness(x, ln, block=BLOCK, curves=True, groups=GROUPS)),
    ("dr14", lambda x, ln: B.programme_dr14(x, ln, block=BLOCK, curves=True, groups=GROUPS)),
    ("truepeak", lambda x, ln: B.programme_truepeak(x, ln, block=BLOCK, groups=GROUPS)),
    ("needle_vu", lambda x, ln: B.programme_needle(x, ln, B.PPM_VU, block=BLOCK, groups=GROUPS)),
    ("needle_ms", lambda x, ln: B.programme_needle(x, ln, B.PPM_MS, block=BLOCK, groups=GROUPS)),
    ("correlation", lambda x, ln: B.programme_correlation(x, ln, block=BLOCK, groups=GROUPS)),
    ("spectrum", lambda x, ln: B.programme_spectrum(x, ln, block=BLOCK, groups=GROUPS)),
    ("stereo", lambda x, ln: B.programme_stereo(x, ln, block=BLOCK, groups=GROUPS)),
    ("stats", lambda x, ln: B.programme_stats(x, np.repeat(ln, 2), block=BLOCK)),
])
def test_programme_s16(s16, name, fn):
    a, lengths, host = s16
    same(fn(B.pcm_source(a), lengths), fn(host, lengths))


@pytest.mark.parametrize("nchan", [2, 6])
@pytest.mark.parametrize("fmt", [P.S24, P.S32, P.F32])
def test_programme_wide_formats(fmt, nchan):
    rng = np.random.default_rng(20 + 3 * fmt + nchan)
    n, t = 8, 48000 + 777
    a = clips(rng, fmt, n, t, nchan)
    lengths = rng.integers(1, t, size=n)
    lengths[0] = t
    lengths[lengths % BLOCK == 0] += 1
    host = P.planar(a, fmt)
    gains = B.bs1770_weights([30, -30, 0, 0, 110, -110], [0] * 6) if nchan == 6 else None     # 5.1: L R C LFE Ls Rs
    loud = lambda x: B.programme_loudness(x, lengths, nchan=nchan, gains=gains, block=BLOCK, curves=True)
    tp = lambda x: B.programme_truepeak(x, lengths, nchan=nchan, block=BLOCK)
    same(loud(B.pcm_source(a)), loud(host))
    same(tp(B.pcm_source(a)), tp(host))


def test_programme_on_caller_stream(s16):
    a, lengths, host = s16
    want = B.programme_loudness(host, lengths, block=BLOCK)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = B.programme_loudness(B.pcm_source(a), lengths, block=BLOCK)
    same(got, want)


def test_decoder_fresh_blocks(s16):
    """a decoder returns a new array for every block; every block's rows must reach the device as they were at the call, also
    when the uploads queue behind earlier work and the two slots come round again"""
    a, lengths, host = s16
    calls = []

    def decode(off, nfram):
        calls.append((off, nfram))
        return a[:, off:off + nfram].copy()
    f = B.pcm_source(decode, nchan=2, fmt=B.PCM_S16)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)                       # the copies below queue behind this on the stream
    outs = [f(b * BLOCK, BLOCK) for b in range(6)]
    torch.cuda.synchronize()
    for b, o in enumerate(outs):
        assert np.array_equal(u32(o), u32(host[:, b * BLOCK:(b + 1) * BLOCK])), b
    calls.clear()
    same(B.programme_loudness(f, lengths, block=BLOCK), B.programme_loudness(host, lengths, block=BLOCK))
    assert len(calls) == -(-int(lengths.max()) // BLOCK) >= 5
