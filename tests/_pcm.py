"""numpy restatement of b200m_pcm_planar_device: interleaved PCM [N, T, nchan] (uint8 [N, T, nchan, 3] for packed 24-bit) to the
planar float32 rows [N * nchan, T], row i * nchan + c = channel c of clip i, scaled by 2^-(bits - 1)."""
import numpy as np

S16, S24, S32, F32 = 0, 1, 2, 3
BYTES = (2, 3, 4, 4)
DTYPE = (np.int16, np.uint8, np.int32, np.float32)


def values(a, fmt):
    """the float32 value of every sample of a, shape a.shape (without the byte axis for S24)"""
    if fmt == S16:
        return a.astype(np.float32) * np.float32(2.0 ** -15)                     # exact
    if fmt == S24:
        u = a[..., 0].astype(np.int32) | a[..., 1].astype(np.int32) << 8 | a[..., 2].astype(np.int32) << 16
        return ((u << 8) >> 8).astype(np.float32) * np.float32(2.0 ** -23)      # sign-extended, exact
    if fmt == S32:
        return a.astype(np.float32) * np.float32(2.0 ** -31)                     # numpy's cast rounds to nearest-even
    return a.view(np.float32).copy()                                             # F32: a bit copy


def planar(a, fmt):
    """float32 [N * nchan, T] of the PCM array a [N, T, nchan(, 3)]"""
    v = values(a, fmt)
    n, t, c = v.shape
    return np.ascontiguousarray(v.transpose(0, 2, 1).reshape(n * c, t))


def raw(a, fmt):
    """a's bytes as uint8 [N, T * nchan * bytes]: the interleaved clips as a file holds them"""
    return np.ascontiguousarray(a).view(np.uint8).reshape(a.shape[0], -1)


def random(rng, n, t, nchan, fmt):
    """PCM [N, T, nchan(, 3)] of random bytes: every bit pattern of the format, for F32 NaN payloads, infinities and denormals"""
    b = rng.integers(0, 256, size=(n, t, nchan, BYTES[fmt]), dtype=np.uint8)
    return b if fmt == S24 else b.view(DTYPE[fmt]).reshape(n, t, nchan)
