"""GPU: album loudness at library scale -- b200m_ebu_group_reduce / b200m_ebu_group_finish on the shapes a library meets.

tests/test_ebu_group_gpu.py checks the album path on 96 instances (at most 6 reduce CTAs) and 40 s of audio.  This file checks it
where its design is stressed: up to 512 CTAs adding into one album row, G up to B200M_MAX_GROUPS, album edges at every position
of a CTA's member chunk and load batch, and block counts at the int32 bound.  The reference for every reduce is the int64 sum of
the bank's own per-instance histograms and count words, read in one b200m_ebu_snapshot; those histograms are anchored on a sample
of instances to private oracle instances fed the same audio.  The reference for every finish is the reference's own
Ebu_r128_hist::calc_integ / calc_range (oracle hist_calc) on the int64 row, compared bit for bit.
 1. the headline bank (8192 stereo EBUr128 instances, tolerance mode: the fused kernel) after 200 blocks of program-like input
    with silent instances and instances clamped at bin 750: G = 1, 64, 1024, 8192, the skewed shape, an album of every 16th
    instance, album sizes cycling 1..33, 1 / 15 / 16 / 17 members in all, and G = 65536 with 300 albums in use;
 2. synthetic histograms written by b200m_ebu_restore: an album at exactly 2^31 - 1 M-blocks, S counts between 2^24 and 2^30;
 3. host-side state: d_out at a 4-byte offset between sentinel rows, the member-list cache, the finish's result buffer growing and
    being reused, and two shard banks summing to the full bank;
 4. programme_loudness(..., groups=...) on 256 clips of 1-20 s in 40 albums against private oracle instances.
"""
import types

import numpy as np
import pytest
import scipy.sparse as sp

import _oracle as O
from test_ebu_gating_gpu import Program, hist_families, mix_vector

pytestmark = pytest.mark.gpu
FS = 48000.0
MIX = 1508
HIST_PITCH = 752          # int32 words per instance histogram (751 bins and a zero pad word), csrc/ebu.cu
GRP_CHUNK = 16            # members per ebu_group_reduce_kernel CTA, csrc/ebu.cu
GRP_BATCH = 4             # members per load batch of that kernel
N = 8192                  # bench.py's headline bank
BLOCKS = 200
I32_MAX = 2 ** 31 - 1


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _pad16(b):
    return (b + 15) & ~15


def snapshot(ebu):
    """b200m_ebu_snapshot of an EBU bank as a writable uint8 blob"""
    import meters_lv2_b200 as B
    L = B.lib()
    size = L.b200m_ebu_snapshot_size(ebu.h)
    buf = np.empty(size, np.uint8)
    B._ck(L.b200m_ebu_snapshot(ebu.h, B._np_ptr(buf), size, B._stream_ptr(None)))
    return buf


def restore(ebu, buf):
    import meters_lv2_b200 as B
    B._ck(B.lib().b200m_ebu_restore(ebu.h, B._np_ptr(buf), buf.size, B._stream_ptr(None)))


def hist_views(buf, n):
    """histM [n, HIST_PITCH], histS [n, HIST_PITCH], cnt [n, 4] (int32 views into the blob): the snapshot's last four segments are
    histM, histS, cnt and fph, each padded to 16 bytes, so their offsets follow from the blob's size"""
    hb = HIST_PITCH * 4 * n
    c0 = buf.size - _pad16(4 * n) - _pad16(16 * n)
    s0 = c0 - _pad16(hb)
    m0 = s0 - _pad16(hb)
    hm = buf[m0:m0 + hb].view(np.int32).reshape(n, HIST_PITCH)
    hs = buf[s0:s0 + hb].view(np.int32).reshape(n, HIST_PITCH)
    cnt = buf[c0:c0 + 16 * n].view(np.int32).reshape(n, 4)
    return hm, hs, cnt


def mix_rows(buf, n):
    """int64 [n, MIX]: every instance's histograms and count words in the b200m_ebu_mix_reduce layout"""
    hm, hs, cnt = hist_views(buf, n)
    assert not hm[:, 751].any() and not hs[:, 751].any()
    return np.concatenate([hm, hs, cnt], axis=1).astype(np.int64)


def album_sums(V, groups, G):
    """int64 [G, MIX]: the rows of V summed per album (group -1: in no album)"""
    groups = np.asarray(groups, np.int64)
    m = np.nonzero(groups >= 0)[0]
    S = sp.csr_matrix((np.ones(m.size, np.int64), (groups[m], m)), shape=(G, V.shape[0]))
    return np.asarray(S @ V)


def oracle_finish(rows):
    return np.stack([O.hist_calc(r[:751], int(r[1504]), r[752:1503], int(r[1505])) for r in rows])


def reduce_and_check(ebu, V, groups, G, garbage=-3):
    """group_reduce into rows holding garbage, then: rows == int64 sums, finish == hist_calc, empty albums -200.
    -> (rows int64 [G, MIX], finish float32 [G, 5])"""
    import torch
    d = torch.full((G, MIX), garbage, dtype=torch.int32, device="cuda")
    ebu.group_reduce(groups, d)
    want = album_sums(V, groups, G)
    assert want.min() >= 0 and want.max() <= I32_MAX
    got = d.cpu().numpy().astype(np.int64)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, ("rows differ", G, bad[:8])
    fin = ebu.group_finish(d)
    assert fin.shape == (G, 5)
    bad = np.nonzero((u32(fin) != u32(oracle_finish(want))).any(axis=1))[0]
    assert bad.size == 0, ("finish differs", G, bad[:8])
    empty = np.setdiff1d(np.arange(G), groups)
    assert (fin[empty] == -200.0).all()
    return want, fin


def member_starts(groups, G):
    """start of each non-empty album in the reduce's member list (instances sorted by album)"""
    sizes = np.bincount(np.asarray(groups)[np.asarray(groups) >= 0], minlength=G)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    return starts[sizes > 0]


# ---------------------------------------------------------------------------------------------- 1. the headline bank
@pytest.fixture(scope="module")
def headline():
    """8192 stereo EBUr128 instances in tolerance mode and two 4096-instance shard banks over the same rows, after 200 blocks of
    1024 frames: instance i plays Program instance i % 512 at its own gain (instances 0..511 at 0 dB: instance 0 is the Tech 3341
    tone), some are silent, some play uniform noise peaking at +18 dBFS (every M block clamped at bin 750).  A private oracle of 32
    instances is fed the same rows.  -> namespace(bank, shards, V [N, MIX] int64 from one snapshot, silent, loud)"""
    import torch
    import meters_lv2_b200 as B
    from meters_lv2_b200 import shard
    rng = np.random.default_rng(8192)
    base = Program(512, 2, seed=8192)
    gain_db = rng.uniform(-30.0, 6.0, N)
    gain_db[:512] = 0.0
    silent = np.sort(rng.choice(np.arange(512, N), 12, replace=False))
    loud = np.sort(rng.choice(np.setdiff1d(np.arange(512, N), silent), 12, replace=False))
    gain = 10.0 ** (gain_db / 20.0)
    gain[silent] = 0.0
    gain_d = torch.from_numpy(np.repeat(gain, 2).astype(np.float32)).cuda()[:, None]
    src = torch.from_numpy(np.repeat(2 * (np.arange(N) % 512), 2) + np.tile([0, 1], N)).cuda()
    loud_rows = torch.from_numpy(np.stack([2 * loud, 2 * loud + 1], axis=1).ravel()).cuda()
    sample = np.unique(np.concatenate([[0, 1, 2, 3, N - 1], silent[:3], loud[:3], rng.choice(N, 19, replace=False)]))[:32]
    sample_rows = torch.from_numpy(np.stack([2 * sample, 2 * sample + 1], axis=1).ravel()).cuda()
    noise = torch.Generator(device="cuda"); noise.manual_seed(8192)

    bank = B.EBUr128(N, FS, True); bank.set_precision(B.PREC_FMA)
    exact = B.EBUr128(N, FS, True)
    shards = []
    for r in range(2):
        lo, cnt = shard.shard_range(N, r, 2)
        b = B.EBUr128(cnt, FS, True); b.set_precision(B.PREC_FMA); shards.append((lo, cnt, b))
    for b in (bank, exact, *(s[2] for s in shards)):
        b.control(B.EBUr128.START)
    o = O.Ebu(sample.size, 2); o.integr("start")
    for blk in range(BLOCKS):
        xs = torch.from_numpy(base.next(1024)).cuda()
        xd = xs[src] * gain_d
        xd[loud_rows] = (torch.rand((loud_rows.numel(), 1024), device="cuda", generator=noise) * 2 - 1) * 8.0
        if blk < 3:
            # the fused kernel runs: the exact bank's K1 + true-peak FIR pair is one kernel in the tolerance-mode bank
            torch.cuda.synchronize()
            l0 = B.launch_count(); bank.run(xd); torch.cuda.synchronize(); lf = B.launch_count() - l0
            l0 = B.launch_count(); exact.run(xd); torch.cuda.synchronize(); le = B.launch_count() - l0
            assert le - lf == 1, (blk, lf, le)
        else:
            bank.run(xd)
        for lo, cnt, b in shards:
            b.run(xd[2 * lo:2 * (lo + cnt)])
        o.process(np.ascontiguousarray(xd[sample_rows].cpu().numpy()), nthreads=8)
    exact.close()
    torch.cuda.synchronize()
    V = mix_rows(snapshot(bank.ebu), N)
    for k, i in enumerate(sample):
        hm, hs, c = o.hist(k)
        assert np.array_equal(V[i, :751], hm) and np.array_equal(V[i, 752:1503], hs) and np.array_equal(V[i, 1504:], c), i
    assert not V[silent].any()
    assert (V[loud, 1506] == V[loud, 1504]).all() and (V[loud, 1504] > 30).all()       # every block of a loud instance clamps
    assert (V[loud, 750] == V[loud, 1504]).all()
    assert (V[:, 1504] > 0).sum() > 0.9 * N                  # the rest stayed below the -70 LUFS gate
    return types.SimpleNamespace(bank=bank, shards=shards, V=V, silent=silent, loud=loud)


def _cycling_sizes(n, rng):
    """album sizes 1, 2, .., 33, 1, 2, .. over a permutation of the instances (the last album cut short)"""
    perm = rng.permutation(n)
    g = np.empty(n, np.int64)
    pos, a = 0, 0
    while pos < n:
        s = min(1 + a % 33, n - pos)
        g[perm[pos:pos + s]] = a
        pos += s; a += 1
    return g, a


def _few_members(n, rng, sizes):
    """sum(sizes) instances in albums of the given sizes (album k holds sizes[k] random instances), every other instance in none"""
    g = np.full(n, -1, np.int64)
    pick = rng.choice(n, sum(sizes), replace=False)
    g[pick] = np.repeat(np.arange(len(sizes)), sizes)
    return g, len(sizes) + 2                                  # two empty albums after the last


def _assignments(n, seed):
    rng = np.random.default_rng(seed)
    half = n // 2
    perm = rng.permutation(n)
    skew = np.empty(n, np.int64)
    skew[perm[:half]] = 0
    skew[perm[half:]] = 1 + np.arange(n - half)
    every16 = rng.integers(0, 10, n)
    every16[every16 == 5] = 6
    every16[::16] = 5
    g64 = rng.integers(-1, 64, n)
    out = {"G=1": (np.zeros(n, np.int64), 1),
           "G=64 with unassigned": (g64, 64),
           "G=1024": (rng.integers(0, 1024, n), 1024),
           "G=8192 permuted": (rng.permutation(n), n),
           "skewed": (skew, 1 + n - half),
           "every 16th": (every16, 10),
           "sizes 1..33": _cycling_sizes(n, rng)}
    for sizes in ([1], [4, 1, 10], [16], [5, 11, 1]):          # 1, 15, 16, 17 members
        out["%d members" % sum(sizes)] = _few_members(n, rng, sizes)
    return out


def test_headline_bank_albums(headline):
    """every assignment: rows = int64 sums, finish = hist_calc, empty albums -200; albums plus unassigned instances = mix_reduce"""
    import torch
    ebu, V = headline.bank.ebu, headline.V
    mix = torch.zeros(MIX, dtype=torch.int32, device="cuda")
    ebu.mix_reduce(mix)
    mix = mix.cpu().numpy().astype(np.int64)
    assert np.array_equal(mix, V.sum(axis=0))
    cases = _assignments(N, seed=1)
    # the shapes reach what they are meant to
    assert (cases["G=1"][0] == 0).sum() // GRP_CHUNK == 512                      # 512 CTAs add into one row
    assert (cases["skewed"][0] == 0).sum() // GRP_CHUNK == 256
    assert np.array_equal(np.nonzero(cases["every 16th"][0] == 5)[0], np.arange(0, N, 16))
    st = member_starts(*cases["sizes 1..33"])
    assert set(st % GRP_CHUNK) == set(range(GRP_CHUNK)) and set(st % GRP_BATCH) == set(range(GRP_BATCH))
    assert [(g >= 0).sum() for k, (g, _) in cases.items() if k.endswith("members")] == [1, 15, 16, 17]
    for name, (groups, G) in cases.items():
        want, fin = reduce_and_check(ebu, V, groups, G)
        assert np.array_equal(want.sum(axis=0) + V[groups < 0].sum(axis=0), mix), name
        if name in ("G=1", "skewed"):
            assert (fin[0, :4] > -100).all(), name                                # gated and ranged: the album is live


def test_headline_bank_max_groups(headline):
    """G = B200M_MAX_GROUPS (395 MB of rows), 300 albums in use, among them the first and the last: the used rows equal the sums,
    every other row is zero and finishes to -200"""
    import torch
    import meters_lv2_b200 as B
    ebu, V = headline.bank.ebu, headline.V
    G = B.MAX_GROUPS
    assert G == 65536
    rng = np.random.default_rng(65536)
    used = np.sort(np.concatenate([[0, G - 1], rng.choice(np.arange(1, G - 1), 298, replace=False)]))
    k = rng.integers(0, used.size, N)
    k[:used.size] = np.arange(used.size)                      # every used album has a member
    groups = used[k]
    d = torch.full((G, MIX), -3, dtype=torch.int32, device="cuda")
    try:
        ebu.group_reduce(groups, d)
        want = album_sums(V, k, used.size)
        nonzero = (d != 0).any(dim=1).cpu().numpy()
        assert np.array_equal(np.nonzero(nonzero)[0], used[want.any(axis=1)])
        assert np.array_equal(d[torch.from_numpy(used).cuda()].cpu().numpy().astype(np.int64), want)
        fin = ebu.group_finish(d)
        assert fin.shape == (G, 5)
        assert np.array_equal(u32(fin[used]), u32(oracle_finish(want)))
        rest = np.setdiff1d(np.arange(G), used)
        assert (fin[rest] == -200.0).all()
    finally:
        del d
        torch.cuda.empty_cache()


def test_shards_sum_to_the_headline_bank(headline):
    """two 4096-instance banks fed the two halves of the headline input, each reduced with its slice of a G = 1024 assignment:
    their summed rows are the full bank's"""
    import torch
    G = 1024
    groups = np.random.default_rng(1024).integers(-1, G, N)
    full = torch.full((G, MIX), 9, dtype=torch.int32, device="cuda")
    headline.bank.ebu.group_reduce(groups, full)
    acc = torch.zeros_like(full)
    for lo, cnt, b in headline.shards:
        d = torch.full_like(full, -9)
        b.ebu.group_reduce(groups[lo:lo + cnt], d)
        acc += d
    assert torch.equal(acc, full)
    assert np.array_equal(full.cpu().numpy().astype(np.int64), album_sums(headline.V, groups, G))


# ---------------------------------------------------------------------------------------------- 2. large block counts
def _split(rng, h, m):
    """int64 [m, 751]: the bins of h split among m members"""
    w = rng.random((m, h.size)) + 0.05
    p = np.floor(w / w.sum(axis=0) * h).astype(np.int64)
    p[0] += h - p.sum(axis=0)
    assert (p >= 0).all()
    return p


def _speech(rng, total, heavy=None):
    """an album histogram of `total` points: a speech-range cluster, clusters near the -10 LU and -20 LU gates below it, bins 0
    and 750, and (heavy) one bin holding all but `heavy` of the points"""
    h = np.zeros(751, np.int64)
    rest = total if heavy is None else heavy
    for lo, hi, share in ((420, 520, 0.6), (330, 390, 0.25), (230, 290, 0.12), (0, 1, 0.02), (750, 751, 0.0002)):
        b = np.arange(lo, hi)
        c = np.floor(rng.random(b.size) / b.size * 1.6 * share * rest).astype(np.int64)
        h[b] += c
    h[470] += rest - h.sum()
    if heavy is not None:
        h[455] += total - heavy
    assert h.sum() == total and (h >= 0).all()
    return h


def test_block_counts_at_the_int32_bound():
    """a 4096-instance bank whose histograms and count words are written by restore: album 0 (512 members) holds exactly
    2^31 - 1 M-blocks, one bin of them within 2^20 of it; albums 1-5 hold 2^24 .. 2^30 S-blocks, albums 6-9 few; some instances
    in no album, albums 10-11 empty.  Rows = int64 sums (each fits int32), finish = hist_calc bit for bit."""
    import meters_lv2_b200 as B
    n, G = 4096, 12
    rng = np.random.default_rng(2 ** 31)
    bank = B.Ebu_r128_proc(n, 2)
    perm = rng.permutation(n)
    groups = np.full(n, -1, np.int64)
    sizes = [512, 300, 300, 300, 300, 300, 100, 50, 17, 1]
    pos = 0
    for a, s in enumerate(sizes):
        groups[perm[pos:pos + s]] = a
        pos += s
    hm = np.zeros((n, 751), np.int64); hs = np.zeros((n, 751), np.int64)
    s_tot = np.exp(rng.uniform(np.log(2 ** 24 + 1), np.log(2 ** 30 - 1), 5)).astype(np.int64)
    s_tot[0] = 2 ** 30 - 1
    for a in range(len(sizes)):
        mem = np.nonzero(groups == a)[0]
        if a == 0:
            am, as_ = _speech(rng, I32_MAX, heavy=int(rng.integers(2 ** 16, 2 ** 20))), _speech(rng, 2 ** 22)
        elif a <= 5:
            am, as_ = _speech(rng, int(rng.integers(2 ** 20, 2 ** 28))), _speech(rng, int(s_tot[a - 1]))
        else:
            am, as_ = _speech(rng, int(rng.integers(40, 4000))), _speech(rng, int(rng.integers(15, 400)))
        hm[mem] = _split(rng, am, mem.size); hs[mem] = _split(rng, as_, mem.size)
    out = np.nonzero(groups < 0)[0]
    hm[out] = rng.integers(0, 1000, (out.size, 751)); hs[out] = rng.integers(0, 100, (out.size, 751))
    buf = snapshot(bank)
    vm, vs, vc = hist_views(buf, n)
    assert np.abs(hm).max() <= I32_MAX and np.abs(hs).max() <= I32_MAX
    vm[:, :751] = hm; vs[:, :751] = hs
    vc[:, 0] = hm.sum(axis=1); vc[:, 1] = hs.sum(axis=1)
    vc[:, 2] = rng.integers(1, 4, n); vc[:, 3] = rng.integers(1, 4, n)                  # the clamp counts: summed, not gated
    restore(bank, buf)
    V = mix_rows(snapshot(bank), n)
    assert np.array_equal(V[:, :751], hm) and np.array_equal(V[:, 752:1503], hs)
    want, fin = reduce_and_check(bank, V, groups, G)
    # the run reaches what it claims: exactly 2^31 - 1 M-blocks, a bin near it, S counts above 2^24
    assert want[0, 1504] == I32_MAX and want[0, :751].max() >= I32_MAX - 2 ** 20
    assert (want[1:6, 1505] > 2 ** 24).all() and (want[1:6, 1505] < 2 ** 30).all() and want[1, 1505] == 2 ** 30 - 1
    assert not want[10:].any()
    assert (fin[:6, :4] > -100).all()
    # the same histograms, the 2^31 - 1 album after another one in the member list
    g2 = np.full(n, -1, np.int64)
    g2[groups == 0] = 1
    g2[(groups == 1) | (groups >= 6)] = 0
    reduce_and_check(bank, V, g2, 2)


# ---------------------------------------------------------------------------------------------- 3. host-side state
@pytest.fixture(scope="module")
def small():
    """a 2048-instance EBU bank fed 12 s of noise at a level per instance and block; `feed` adds more"""
    import torch
    import meters_lv2_b200 as B
    n = 2048
    bank = B.Ebu_r128_proc(n, 2); bank.integr_start()
    gen = torch.Generator(device="cuda"); gen.manual_seed(2048)

    def feed(blocks):
        for _ in range(blocks):
            lvl = 10.0 ** (torch.rand(n, 1, device="cuda", generator=gen) * -3.0)
            x = (torch.rand(2 * n, 1024, device="cuda", generator=gen) * 2 - 1) * lvl.repeat_interleave(2, 0)
            bank.process(x)
        torch.cuda.synchronize()
        return mix_rows(snapshot(bank), n)
    return types.SimpleNamespace(n=n, bank=bank, feed=feed, V=feed(560))


def test_output_rows_at_an_unaligned_offset(small):
    """d_out one word past a sentinel row inside a buffer of garbage: the G rows are zeroed and summed, the sentinels untouched"""
    import torch
    n, bank = small.n, small.bank
    V = small.feed(0)
    G = 37
    groups = np.random.default_rng(37).integers(-1, G, n)
    groups[groups == 36] = 35                                 # album 36 empty: its garbage must be zeroed too
    gen = torch.Generator(device="cuda"); gen.manual_seed(37)
    buf = torch.randint(-2 ** 31, 2 ** 31 - 1, ((G + 2) * MIX + 1,), dtype=torch.int32, device="cuda", generator=gen)
    keep = buf.clone()
    lo = MIX + 1
    d = buf[lo:lo + G * MIX].view(G, MIX)
    assert d.data_ptr() % 16 == 4 and d.is_contiguous()
    bank.group_reduce(groups, d)
    assert torch.equal(buf[:lo], keep[:lo]) and torch.equal(buf[lo + G * MIX:], keep[lo + G * MIX:])
    want = album_sums(V, groups, G)
    assert np.array_equal(d.cpu().numpy().astype(np.int64), want)
    assert np.array_equal(u32(bank.group_finish(d)), u32(oracle_finish(want)))
    assert torch.equal(buf[:lo], keep[:lo]) and torch.equal(buf[lo + G * MIX:], keep[lo + G * MIX:])


def test_member_list_cache(small):
    """assignment A, more audio, A again (the rows follow the new histograms); A with only the last entry changed, with only the
    first changed, A with a larger G: each reduce matches its own assignment"""
    n, bank = small.n, small.bank
    rng = np.random.default_rng(50)
    G = 50
    A = rng.integers(0, G, n)
    reduce_and_check(bank, small.feed(0), A.copy(), G)
    V = small.feed(40)
    reduce_and_check(bank, V, A.copy(), G)
    assert V[n - 1, 1504] > 0 and V[0, 1504] > 0
    last = A.copy(); last[-1] = (A[-1] + 1) % G
    reduce_and_check(bank, V, last, G)
    first = A.copy(); first[0] = (A[0] + 7) % G
    reduce_and_check(bank, V, first, G)
    reduce_and_check(bank, V, A.copy(), G + 13)


def test_finish_result_buffer_grows_and_is_reused(small):
    """group_finish on rows written by torch (synthetic histograms of every gating family) with G = 5, 65536, 3, 8192: the
    result buffer grows once and is reused at smaller sizes; every result equals hist_calc"""
    import torch
    import meters_lv2_b200 as B
    pool = np.stack([mix_vector(hm, hs) for _, hm, hs in hist_families(n_per_family=24, seed=77)])
    pool = np.concatenate([pool, np.zeros((1, MIX), np.int32)])
    pool_fin = oracle_finish(pool.astype(np.int64))
    pool_d = torch.from_numpy(pool).cuda()
    rng = np.random.default_rng(5)
    for G in (5, B.MAX_GROUPS, 3, 8192):
        k = rng.integers(0, pool.shape[0], G)
        k[:min(G, 3)] = [pool.shape[0] - 1, 0, 1][:min(G, 3)]
        d = pool_d[torch.from_numpy(k).cuda()].contiguous()
        fin = small.bank.group_finish(d)
        assert fin.shape == (G, 5)
        bad = np.nonzero((u32(fin) != u32(pool_fin[k])).any(axis=1))[0]
        assert bad.size == 0, (G, bad[:8])
        del d
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- 4. programme_loudness albums
class _Clips:
    """256 stereo clips, block b (1024 frames) generated from (seed, b) alone: uniform noise at a level per clip and per 0.5 s
    segment, -70 .. 0 dBFS or silence, so the relative gates remove whole segments"""

    def __init__(self, n, seed):
        rng = np.random.default_rng(seed)
        self.n, self.seed = n, seed
        lv = rng.choice([-70.0, -45.0, -35.0, -28.0, -23.0, -18.0, -12.0, -6.0, 0.0, -np.inf], size=(n, 64))
        self.gain = np.repeat(10.0 ** (lv / 20.0), 2, axis=0).astype(np.float32)

    def __call__(self, off, nfram):
        b = off // 1024
        rng = np.random.Generator(np.random.Philox(key=self.seed, counter=[0, 0, b, 0]))
        x = rng.random((2 * self.n, nfram), dtype=np.float32) * np.float32(2.0) - np.float32(1.0)
        seg = (off + np.arange(nfram)) // 24000 % 64
        return np.ascontiguousarray(x * self.gain[:, seg])


def test_programme_loudness_albums_at_scale():
    """256 clips of 1-20 s in 40 albums (albums 7, 19 and 33 empty, 9 clips in none): album gated fields = hist_calc on the int64
    sums of private oracle instances' histograms, each fed its clip in the same blocks; album maxima = the members' maxima;
    album_n_clips"""
    import meters_lv2_b200 as B
    n, G, block = 256, 40, 1024
    rng = np.random.default_rng(256)
    ln = rng.integers(int(1 * FS), int(20 * FS) + 1, n)
    groups = rng.choice(np.setdiff1d(np.arange(G), [7, 19, 33]), n)
    groups[rng.choice(n, 9, replace=False)] = -1
    clips = _Clips(n, seed=256)
    out = B.programme_loudness(clips, ln, FS, block=block, groups=groups)
    assert np.array_equal(out["album_n_clips"], np.bincount(groups[groups >= 0], minlength=G))
    for k, empty in (("maxloudn_M", -200.0), ("maxloudn_S", -200.0), ("tp_max", -np.inf)):
        want = np.array([out[k][groups == a].max() if (groups == a).any() else np.float32(empty) for a in range(G)], np.float32)
        assert np.array_equal(u32(out["album_" + k]), u32(want)), k
    orc = [O.Ebu(1, 2) for _ in range(n)]
    for o in orc:
        o.integr("start")
    for off in range(0, int(ln.max()), block):
        nf = min(block, int(ln.max()) - off)
        x = clips(off, nf)
        for i in np.nonzero(ln > off)[0]:
            m = min(nf, int(ln[i]) - off)
            orc[i].process(np.ascontiguousarray(x[2 * i:2 * i + 2, :m]))
    rows = np.zeros((G, MIX), np.int64)
    for i, o in enumerate(orc):
        assert u32(o.read()[0, 4]) == u32(out["integrated"][i]), i
        if groups[i] >= 0:
            hm, hs, c = o.hist(0)
            rows[groups[i], :751] += hm; rows[groups[i], 752:1503] += hs; rows[groups[i], 1504:1508] += c
    fin = oracle_finish(rows)
    for j, k in enumerate(("integrated", "integ_thr", "range_min", "range_max")):
        assert np.array_equal(u32(out["album_" + k]), u32(fin[:, j])), k
    used = np.unique(groups[groups >= 0])
    assert (out["album_integrated"][used] > -100).all() and (out["album_range_max"][used] > -100).all()
    assert (out["album_integrated"][[7, 19, 33]] == -200.0).all()
