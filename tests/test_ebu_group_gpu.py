"""GPU: album loudness -- the grouped histogram reduce and the batched finish (b200m_ebu_group_reduce / b200m_ebu_group_finish).

An album's histograms are the int32 sum of its members' hist_M / hist_S and count words (the b200m_ebu_mix_reduce layout, one row
per album), and its gated statistics are the reference's Ebu_r128_hist::calc_integ / calc_range on that sum (oracle hist_calc).
Checked here:
 1. a bank of 96 stereo instances against the oracle after 40 s of program-like input in blocks of mixed sizes, reaching the
    bin-750 clamp: every album row equals the int64 sum of its members' oracle histograms and counts, every finish equals
    hist_calc bit for bit, for an assignment with empty albums, one album of more than half the bank, singletons and instances
    in no album;
 2. one album of the whole bank is the whole mix; no instance in any album gives zero rows; one album per instance;
 3. three shard banks reduced with the same G sum to the single bank's rows;
 4. an EBUr128 bank's EBU bank on the host path and on the device path with a caller stream, the assignment changing between
    calls (the cached member list);
 5. programme_loudness(groups=...) against private oracle instances of each clip, summed by album;
 6. argument errors: codes, nothing enqueued.
"""
import numpy as np
import pytest

import _oracle as O
from test_ebu_gating_gpu import Program, ragged_blocks

pytestmark = pytest.mark.gpu
FS = 48000.0
MIX = 1508


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def oracle_rows(o, groups, n_groups):
    """int64 [n_groups, MIX]: the members' oracle histograms and count words summed per album"""
    rows = np.zeros((n_groups, MIX), np.int64)
    for i, g in enumerate(groups):
        if g >= 0:
            hm, hs, c = o.hist(i)
            rows[g, :751] += hm; rows[g, 752:1503] += hs; rows[g, 1504:1508] += c
    return rows


def oracle_finish(rows):
    return np.stack([O.hist_calc(r[:751], int(r[1504]), r[752:1503], int(r[1505])) for r in rows])


def album_assignment(n, seed):
    """37 albums over n instances: album 3 holds more than half the bank, albums 10-17 one instance each, the rest spread
    over albums 20-35 with some left empty, six instances in no album"""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n)
    g = np.full(n, -1, np.int64)
    big = n // 2 + 2
    g[perm[:big]] = 3
    g[perm[big:big + 8]] = np.arange(10, 18)
    rest = perm[big + 8:n - 6]
    g[rest] = rng.choice([20, 21, 23, 24, 27, 30, 31, 35], size=rest.size)
    return g, 37


@pytest.fixture(scope="module")
def driven():
    """a bank of 96 stereo instances, three shard banks over the same rows and the oracle, after 40 s of program-like input"""
    import torch
    import meters_lv2_b200 as B
    from meters_lv2_b200 import shard
    n = 96
    gen = Program(n, 2, seed=9600)
    full = B.Ebu_r128_proc(n, 2); full.integr_start()
    parts = []
    for r in range(3):
        lo, cnt = shard.shard_range(n, r, 3)
        b = B.Ebu_r128_proc(cnt, 2); b.integr_start(); parts.append((lo, cnt, b))
    o = O.Ebu(n, 2); o.integr("start")
    for nf in ragged_blocks(40.0, seed=96):
        x = gen.next(nf)
        xd = torch.from_numpy(x).cuda()
        full.process(xd)
        for lo, cnt, b in parts:
            b.process(xd[2 * lo:2 * (lo + cnt)])
        o.process(x, nthreads=8)
    torch.cuda.synchronize()
    return n, full, parts, o


def test_group_rows_and_finish_equal_oracle(driven):
    import torch
    n, bank, _, o = driven
    groups, G = album_assignment(n, seed=1)
    d = torch.full((G, MIX), 7, dtype=torch.int32, device="cuda")          # the reduce zeroes the rows itself
    bank.group_reduce(groups, d)
    got = d.cpu().numpy()
    want = oracle_rows(o, groups, G)
    assert want.max() < 2 ** 31
    assert np.array_equal(got.astype(np.int64), want)
    # the run reaches what it is meant to: the bin-750 clamp (error words), empty albums, albums above both gating thresholds
    assert want[3, 1506] > 0 and want[3, 1507] > 0
    empty = np.setdiff1d(np.arange(G), groups)
    assert empty.size >= 10 and not want[empty].any()
    assert (want[:, 1504] >= 50).sum() >= 10 and (want[:, 1505] >= 20).sum() >= 10
    fin = bank.group_finish(d)
    assert fin.shape == (G, 5)
    assert np.array_equal(u32(fin), u32(oracle_finish(want)))
    assert (fin[empty] == -200.0).all()
    assert (fin[3] > -100).all()


def test_one_album_is_the_whole_mix_and_no_album_is_zero(driven):
    import torch
    import meters_lv2_b200 as B
    n, bank, _, o = driven
    mix = torch.zeros(B.MIX_WORDS, dtype=torch.int32, device="cuda")
    bank.mix_reduce(mix)
    d = torch.full((1, MIX), -5, dtype=torch.int32, device="cuda")
    bank.group_reduce(np.zeros(n, np.int64), d)
    assert torch.equal(d[0], mix)
    assert np.array_equal(u32(bank.group_finish(d)[0]), u32(bank.mix_finish(mix)))
    # every instance in no album: G rows of zeros, each finishing to "nothing"
    d = torch.full((5, MIX), 3, dtype=torch.int32, device="cuda")
    bank.group_reduce(np.full(n, -1), d)
    assert not d.any().item()
    assert (bank.group_finish(d) == -200.0).all()
    # one album per instance, and more albums than instances: each row is that instance's histograms
    G = n + 9
    d = torch.full((G, MIX), 1, dtype=torch.int32, device="cuda")
    groups = np.random.default_rng(2).permutation(G)[:n]
    bank.group_reduce(groups, d)
    want = oracle_rows(o, groups, G)
    assert np.array_equal(d.cpu().numpy().astype(np.int64), want)
    assert np.array_equal(u32(bank.group_finish(d)), u32(oracle_finish(want)))


def test_shards_sum_to_the_single_bank(driven):
    import torch
    n, bank, parts, _ = driven
    groups, G = album_assignment(n, seed=3)
    full = torch.empty((G, MIX), dtype=torch.int32, device="cuda")
    bank.group_reduce(groups, full)
    acc = torch.zeros_like(full)
    for lo, cnt, b in parts:
        d = torch.empty_like(full)
        b.group_reduce(groups[lo:lo + cnt], d)                  # a shard may hold no member of many albums: the same G
        acc += d
    assert torch.equal(acc, full)
    assert np.array_equal(u32(parts[1][2].group_finish(acc)), u32(bank.group_finish(full)))


def test_r128_host_and_device_path_with_changing_assignment():
    """the EBU bank of two EBUr128 banks, one fed numpy blocks (host path), one CUDA blocks on a caller stream (device path);
    between blocks the album assignment cycles A, A, B, C, A, ...: each reduce matches the oracle sums for the assignment of that
    call, on both paths, and both finish the same"""
    import torch
    import meters_lv2_b200 as B
    n = 40
    gen = Program(n, 2, seed=4000)
    host, dev = B.EBUr128(n, FS, True), B.EBUr128(n, FS, True)
    for b in (host, dev):
        b.control(B.EBUr128.START)
    o = O.Ebu(n, 2); o.integr("start")
    rng = np.random.default_rng(40)
    assign = [(rng.integers(-1, 6, size=n), 6), (rng.integers(0, 3, size=n), 3), (np.arange(n) % 11, 13)]
    order = [0, 0, 1, 2, 0, 2, 2, 1]
    st = torch.cuda.Stream()
    k = 0
    for bi, nf in enumerate(ragged_blocks(16.0, seed=41)):
        x = gen.next(nf)
        host.run(x)
        with torch.cuda.stream(st):
            xd = torch.from_numpy(x).to("cuda", non_blocking=False)
        st.synchronize()
        dev.run(xd, stream=st)
        o.process(x, nthreads=8)
        if bi % 40 != 39:
            continue
        groups, G = assign[order[k % len(order)]]
        k += 1
        torch.cuda.synchronize()
        dh = torch.empty((G, MIX), dtype=torch.int32, device="cuda")
        dd = torch.empty((G, MIX), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        host.ebu.group_reduce(groups, dh)                     # on the bank's own stream: the host path's
        dev.ebu.group_reduce(groups, dd, stream=st)
        st.synchronize(); torch.cuda.synchronize()
        want = oracle_rows(o, groups, G)
        assert np.array_equal(dh.cpu().numpy().astype(np.int64), want), (bi, k)
        assert np.array_equal(dd.cpu().numpy().astype(np.int64), want), (bi, k)
        fh, fd = host.ebu.group_finish(dh), dev.ebu.group_finish(dd, stream=st)
        assert np.array_equal(u32(fh), u32(fd)) and np.array_equal(u32(fh), u32(oracle_finish(want))), (bi, k)
    assert k >= len(order)


def test_programme_loudness_albums():
    """clips of different lengths in albums (one empty, two clips in none): per-clip fields and curves bit-identical to the call
    without groups; album maxima the members' maxima; album gated fields = hist_calc on the sum of private oracle instances'
    histograms, each fed its clip in the same blocks"""
    import meters_lv2_b200 as B
    fs, block, n = 48000.0, 1024, 14
    rng = np.random.default_rng(14)
    ln = rng.integers(int(0.5 * fs), int(14 * fs), size=n)
    ln[5] = 0
    x = Program(n, 2, seed=1400).next(int(ln.max()))
    groups = np.array([0, 0, 2, 2, 2, 2, -1, 3, 0, 4, 4, -1, 3, 2])          # album 1 is empty; clip 5 is empty
    G = 5
    plain = B.programme_loudness(x, ln, fs, block=block, curves=True)
    out = B.programme_loudness(x, ln, fs, block=block, curves=True, groups=groups)
    for k, v in plain.items():
        assert out[k].dtype == v.dtype and out[k].tobytes() == v.tobytes(), k
    for k in ("album_integrated", "album_integ_thr", "album_range_min", "album_range_max", "album_maxloudn_M", "album_maxloudn_S",
              "album_tp_max"):
        assert out[k].shape == (G,) and out[k].dtype == np.float32, k
    assert np.array_equal(out["album_n_clips"], [3, 0, 5, 2, 2]) and out["album_n_clips"].dtype == np.int64
    for a in range(G):
        m = groups == a
        for k, empty in (("maxloudn_M", -200.0), ("maxloudn_S", -200.0), ("tp_max", -np.inf)):
            want = plain[k][m].max() if m.any() else np.float32(empty)
            assert u32(out["album_" + k][a]) == u32(want), (a, k)
    rows = np.zeros((G, MIX), np.int64)
    for i in range(n):
        o = O.Ebu(1, 2); o.integr("start")
        for off in range(0, int(ln[i]), block):
            o.process(np.ascontiguousarray(x[2 * i:2 * i + 2, off:off + min(block, int(ln[i]) - off)]))
        assert u32(o.read()[0, 4]) == u32(plain["integrated"][i]), i
        if groups[i] >= 0:
            hm, hs, c = o.hist(0)
            rows[groups[i], :751] += hm; rows[groups[i], 752:1503] += hs; rows[groups[i], 1504:1508] += c
    fin = oracle_finish(rows)
    for j, k in enumerate(("integrated", "integ_thr", "range_min", "range_max")):
        assert np.array_equal(u32(out["album_" + k]), u32(fin[:, j])), k
    assert out["album_integrated"][1] == -200.0 and out["album_tp_max"][1] == -np.inf
    assert (out["album_integrated"][[0, 2]] > -100).all()
    # every clip in no album: G = 0
    none = B.programme_loudness(x[:4], ln[:2], fs, block=block, groups=[-1, -1])
    assert none["album_integrated"].shape == (0,) and none["album_n_clips"].shape == (0,)


def test_argument_errors_enqueue_nothing():
    import ctypes as C
    import torch
    import meters_lv2_b200 as B
    L = B.lib()
    bank = B.Ebu_r128_proc(8, 2)
    d = torch.full((4, MIX), 7, dtype=torch.int32, device="cuda")
    dp = C.c_void_p(d.data_ptr())
    out = np.zeros((B.MAX_GROUPS + 1, 5), np.float32)
    ok = np.array([0, 1, 2, 3, B.NO_GROUP, 0, 0, 0], np.uint32)
    bad = ok.copy(); bad[6] = 4
    torch.cuda.synchronize()
    l0 = B.launch_count()
    P = B._np_ptr
    calls = [L.b200m_ebu_group_reduce(bank.h, P(bad), 4, dp, None),                   # an album id >= n_groups
             L.b200m_ebu_group_reduce(bank.h, P(ok), 0, dp, None),
             L.b200m_ebu_group_reduce(bank.h, P(ok), B.MAX_GROUPS + 1, dp, None),
             L.b200m_ebu_group_reduce(None, P(ok), 4, dp, None),
             L.b200m_ebu_group_reduce(bank.h, None, 4, dp, None),
             L.b200m_ebu_group_reduce(bank.h, P(ok), 4, None, None),
             L.b200m_ebu_group_finish(bank.h, dp, 0, P(out), None),
             L.b200m_ebu_group_finish(bank.h, dp, B.MAX_GROUPS + 1, P(out), None),
             L.b200m_ebu_group_finish(None, dp, 4, P(out), None),
             L.b200m_ebu_group_finish(bank.h, None, 4, P(out), None),
             L.b200m_ebu_group_finish(bank.h, dp, 4, None, None)]
    assert calls == [-1] * len(calls)
    assert B.launch_count() == l0
    torch.cuda.synchronize()
    assert (d == 7).all().item(), "a refused call must not touch d_out"
    with pytest.raises(B.B200MError):
        bank.group_reduce([0, 0, 0, 0, 0, 0, 0, -2], d)
    with pytest.raises(B.B200MError):
        bank.group_reduce(np.zeros(7, np.int64), d)
    with pytest.raises(B.B200MError):
        bank.group_reduce(np.zeros(8, np.int64), d.view(-1))
    # the accepted calls: one launch each
    assert L.b200m_ebu_group_reduce(bank.h, P(ok), 4, dp, None) == 0
    assert L.b200m_ebu_group_finish(bank.h, dp, 4, P(out), None) == 0
    assert B.launch_count() == l0 + 2
    assert (out[:4] == -200.0).all()
