"""GPU: the per-pair hold of the correlation bank (b200m_cor_process_ctl_*).  A bank whose pairs run in a random subset of cycles
must match, bit for bit, one private bank per pair that is called only in that pair's active cycles: the five filter states and
the reading, in both precision modes (one lane per pair in exact mode, one warp per pair in FMA mode, so a pair's arithmetic never
depends on its neighbours).  Held pairs keep their state exactly, whatever their input rows hold; a NULL mask is
b200m_cor_process_host."""
import numpy as np
import pytest

import _signals as S

pytestmark = pytest.mark.gpu
N = 300                                                    # the last warp of the exact-mode kernel is partial (300 = 9 * 32 + 12)
BLOCKS = [1024, 333, 1024, 333, 1024, 333, 1024, 333]


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("path", ["host", "device_unaligned"])
@pytest.mark.parametrize("fma", [False, True])
def test_held_pairs_match_private_banks_run_in_their_active_cycles(fma, path):
    import torch
    import meters_lv2_b200 as B
    mode = B.PREC_FMA if fma else B.PREC_EXACT
    bank = B.Stcorrdsp(N)
    bank.set_precision(mode)
    priv = [B.Stcorrdsp(1) for _ in range(N)]
    for p in priv:
        p.set_precision(mode)
    rng = np.random.default_rng(91 + 2 * fma + (path != "host"))
    x = S.white(2 * N, sum(BLOCKS), seed=93)
    for k in range(N):
        x[2 * k + 1] = np.float32(0.7) * x[2 * k] + np.float32(0.3) * x[2 * k + 1]
    want_res = np.zeros(N, np.float32)
    off = 0
    for b, n in enumerate(BLOCKS):
        run = (rng.random(N) < 0.6).astype(np.uint8)
        if b == 0:
            run[:32] = 0                                   # one warp held entirely
        blk = x[:, off:off + n].copy()
        blk[np.repeat(run == 0, 2)] = np.nan               # a held pair's rows are never read
        before = bank.state()
        before_res = bank.read()
        if path == "host":
            bank.process(blk, run=run)
        else:
            # rows 1025 floats apart: the kernels' unaligned load path
            d = torch.zeros((2 * N, 1025), dtype=torch.float32, device="cuda")
            d[:, :n] = torch.from_numpy(blk)
            bank.process(d[:, :n], run=run)
            torch.cuda.synchronize()
        for k in np.flatnonzero(run):
            priv[k].process(np.ascontiguousarray(x[2 * k:2 * k + 2, off:off + n]))
            want_res[k] = priv[k].read()[0]
        got = bank.state()
        got_res = bank.read()
        want = np.concatenate([p.state() for p in priv])
        held = run == 0
        assert np.array_equal(u32(got[held]), u32(before[held])), b
        assert np.array_equal(u32(got_res[held]), u32(before_res[held])), b
        assert np.array_equal(u32(got), u32(want)), (b, np.flatnonzero((u32(got) != u32(want)).any(axis=1))[:8])
        assert np.array_equal(u32(got_res), u32(want_res)), b
        off += n
    assert np.isfinite(bank.state()).all()
    for p in priv + [bank]:
        p.close()


@pytest.mark.parametrize("fma", [False, True])
def test_a_null_or_all_ones_mask_is_the_plain_process_call(fma):
    import meters_lv2_b200 as B
    L = B.lib()
    banks = [B.Stcorrdsp(N) for _ in range(3)]
    for bk in banks:
        bk.set_precision(B.PREC_FMA if fma else B.PREC_EXACT)
    x = S.white(2 * N, 4 * 1024, seed=95)
    ones = np.ones(N, np.uint8)
    for b in range(4):
        blk = np.ascontiguousarray(x[:, b * 1024:(b + 1) * 1024 - 7 * b])
        p, s, n = B._np_ptr(blk), blk.shape[1], blk.shape[1]
        assert L.b200m_cor_process_host(banks[0].h, p, s, n) == 0
        assert L.b200m_cor_process_ctl_host(banks[1].h, p, s, n, None) == 0
        assert L.b200m_cor_process_ctl_host(banks[2].h, p, s, n, B._np_ptr(ones)) == 0
        st = [u32(bk.state()) for bk in banks]
        rd = [u32(bk.read()) for bk in banks]
        assert np.array_equal(st[0], st[1]) and np.array_equal(st[0], st[2]), b
        assert np.array_equal(rd[0], rd[1]) and np.array_equal(rd[0], rd[2]), b
    for bk in banks:
        bk.close()
