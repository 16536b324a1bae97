"""Cost of PCM input (b200m_pcm_planar_device, pcm_source).
  (a) the conversion kernel alone: CUDA-event µs per call over --iters calls after 20 warm-up calls, device-resident input, for
      every format, on 8192 stereo clips x 1024 frames and 2048 stereo clips x 8192 frames, with its rate in GB/s (bytes read +
      bytes written) against the H100 SXM's 3.35 TB/s of HBM3;
  (b) programme_loudness on --clips stereo clips of --blocks blocks of 1024 frames, host-clock ms per block of the whole call (bank
      set-up and results included; a first call of each feed, checked bit for bit against the pinned feed, warms up), fed four ways:
        f32_pinned    a float32 planar array in pinned memory (the bank's host path);
        s16_numpy     int16 interleaved, converted to float32 planar by numpy on the host block by block, then the host path;
        s16_source    pcm_source on the int16 interleaved array;
        s24_source    pcm_source on packed 24-bit interleaved bytes.
Every case is taken --runs times, the case order reversed on every other run.  The GPU's name and power limit are read in the same
call and printed with the results (one JSON line).

    python meters.lv2_b200/host/pcm_cost.py [--iters 200] [--runs 3] [--clips 8192] [--blocks 8]
"""
import ctypes as C
import json

import numpy as np
import torch

import _cost
from _cost import B

KERNEL_SHAPES = ((8192, 1024), (2048, 8192))
FORMATS = (("s16", B.PCM_S16), ("s24", B.PCM_S24), ("s32", B.PCM_S32), ("f32", B.PCM_F32))
HBM_TBS = 3.35


def kernel_cases(a):
    L = B.lib()
    st = B._stream_ptr(None)
    out = {}
    for n, nf in KERNEL_SHAPES:
        for name, fmt in FORMATS:
            bps = B.PCM_BYTES[fmt]
            d_in = torch.randint(0, 256, (n * nf * 2 * bps,), dtype=torch.uint8, device="cuda")
            pitch = (nf + 63) & ~63
            d_out = torch.empty((2 * n, pitch), dtype=torch.float32, device="cuda")
            args = (0, C.c_void_p(d_in.data_ptr()), fmt, n, 2, nf, nf * 2 * bps, C.c_void_p(d_out.data_ptr()), pitch, st)
            us = [_cost.events(lambda: L.b200m_pcm_planar_device(*args), a.iters, 20) for _ in range(a.runs)]
            gbs = [round(n * nf * 2 * (bps + 4) / (u * 1e-6) / 1e9, 1) for u in us]
            out["%dx%d_%s" % (n, nf, name)] = {"us": us, "GB/s": gbs, "of_hbm": [round(g / (HBM_TBS * 1e3), 3) for g in gbs]}
    return out


def programme_cases(a):
    n, nb, blk = a.clips, a.blocks, 1024
    t = nb * blk
    rng = np.random.default_rng(0)
    s16 = rng.integers(-8192, 8192, size=(n, t, 2), dtype=np.int16)
    u = s16.astype(np.int32) << 8                                         # the same audio as packed 24-bit
    s24 = np.stack([u & 0xff, (u >> 8) & 0xff, (u >> 16) & 0xff], axis=-1).astype(np.uint8)
    pinned = B.host_alloc(2 * n, t)
    pinned[:] = (s16.astype(np.float32) * np.float32(2.0 ** -15)).transpose(0, 2, 1).reshape(2 * n, t)
    lengths = np.full(n, t, np.int64)

    def numpy_feed(off, nfram):
        x = s16[:, off:off + nfram].astype(np.float32) * np.float32(2.0 ** -15)
        return np.ascontiguousarray(x.transpose(0, 2, 1).reshape(2 * n, nfram))
    feeds = {"f32_pinned": lambda: pinned, "s16_numpy": lambda: numpy_feed,
             "s16_source": lambda: B.pcm_source(s16), "s24_source": lambda: B.pcm_source(s24)}
    ref = B.programme_loudness(pinned, lengths, block=blk)
    res = {k: [] for k in feeds}
    for r in range(a.runs + 1):                                           # run 0 is the warm-up
        for k in _cost.alternate(feeds, r):
            x = feeds[k]()
            if r == 0:
                got = B.programme_loudness(x, lengths, block=blk)
                assert all(np.array_equal(got[f].view(np.uint32), ref[f].view(np.uint32)) for f in ref), k
            else:
                res[k].append(round(_cost.host_clock(lambda: B.programme_loudness(x, lengths, block=blk)) / 1e3 / nb, 2))
    return {"clips": n, "blocks": nb, "ms_per_block": res}


def main():
    ap = _cost.parser(__doc__, iters=200, runs=3)
    ap.add_argument("--clips", type=int, default=8192, help="stereo clips fed to programme_loudness (default: %(default)s)")
    ap.add_argument("--blocks", type=int, default=8, help="1024-frame blocks per clip (default: %(default)s)")
    a = ap.parse_args()
    gpu = _cost.gpu()
    print(json.dumps({"gpu": gpu, "kernel": kernel_cases(a), "programme_loudness": programme_cases(a)}))


if __name__ == "__main__":
    main()
